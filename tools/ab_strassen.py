"""A/B of the Ozaki-II Strassen route on ONE box, back to back: oz2_strassen 0 (eight residue products per modulus) against 2 (one
Strassen level, seven half-size products, at any eligible size).  python tools/ab_strassen.py [N] [BLK] [REPS] -> one JSON line with the whole-multiply wall
time (context synchronised) and the int8 GEMM launch time (events inside the library) per mode, interleaved 0 / 2 / 0 / 2 so that clock
drift under the power cap hits both alike, the route's counters, and a bit-identity check of sampled output blocks between the modes."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import matrel_b200 as mb  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
blk = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 6
nb = -(-n // blk)
keys = sorted({(0, 0), (nb // 2, nb // 3), (nb - 1, nb - 1), (1, nb - 2), (nb - 1, 0)})
out = {"n": n, "blk": blk, "reps": reps, "blocks_compared": [list(k) for k in keys], "modes": {}}
with mb.MatfastSession(device=0) as s:
    A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
    ref = {}
    for rnd in range(2):
        for mode in (0, 2):
            s.set_option("oz2_strassen", mode)
            s.set_option("time_kernels", 0)
            for _ in range(2):
                C = A.matrixMultiply(n, n, B, n, n, blk)
                del C
            s.sync()
            t0 = time.perf_counter()
            for _ in range(reps):
                C = A.matrixMultiply(n, n, B, n, n, blk)
                del C
            s.sync()
            wall = (time.perf_counter() - t0) / reps * 1e3
            s.set_option("time_kernels", 1)
            s.reset_stats()
            for _ in range(3):
                C = A.matrixMultiply(n, n, B, n, n, blk)
            st = s.stats()
            blocks = [C.get_block(*k).values.copy() for k in keys]
            del C
            ref.setdefault(mode, blocks)
            m = out["modes"].setdefault(str(mode), {"wall_ms": [], "gemm_ms": []})
            m["wall_ms"].append(round(wall, 3))
            m["gemm_ms"].append(round(st["tc_gemm_ms_total"] / 3, 3))
            m["moduli"] = int(st.get("tc_moduli", 0))
            m["tc_int8_ops"] = int(st["tc_int8_ops"])
            m["tc_strassen_jobs"] = int(st["tc_strassen_jobs"])
    out["bit_identical_blocks"] = bool(all(np.array_equal(x, y) for x, y in zip(ref[0], ref[2])))
for k, m in out["modes"].items():
    m["wall_ms_best"] = min(m["wall_ms"])
    m["gemm_ms_best"] = min(m["gemm_ms"])
out["speedup_wall"] = out["modes"]["0"]["wall_ms_best"] / out["modes"]["2"]["wall_ms_best"]
out["speedup_gemm"] = out["modes"]["0"]["gemm_ms_best"] / out["modes"]["2"]["gemm_ms_best"]
out["int8_ops_ratio"] = out["modes"]["2"]["tc_int8_ops"] / out["modes"]["0"]["tc_int8_ops"]
print(json.dumps(out))
