"""A/B of the CTA-pair GEMM's work-item order on ONE box, back to back: oz2_ksplit 0 (modulus, tile pair) against 1 (modulus, K half,
tile pair).  python tools/ab_ksplit.py [N] [BLK] [REPS] -> one JSON line with the whole-multiply wall time (context synchronised) and
the int8 GEMM launch time (events inside the library) per mode, interleaved 0 / 1 / 0 / 1 so that clock drift under the power cap
hits both alike, plus a bit-identity check of one output block between the modes."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import matrel_b200 as mb

n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
blk = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 6
out = {"n": n, "blk": blk, "reps": reps, "modes": {}}
with mb.MatfastSession(device=0) as s:
    A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
    ref = {}
    for rnd in range(2):
        for mode in (0, 1):
            s.set_option("oz2_ksplit", mode)
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
            blk00 = C.get_block(1, 2).values.copy()
            del C
            ref.setdefault(mode, blk00)
            m = out["modes"].setdefault(str(mode), {"wall_ms": [], "gemm_ms": []})
            m["wall_ms"].append(round(wall, 3))
            m["gemm_ms"].append(round(st["tc_gemm_ms_total"] / 3, 3))
            m["moduli"] = int(st.get("tc_moduli", 0))
    out["bit_identical_block"] = bool(np.array_equal(ref[0], ref[1]))
for k, m in out["modes"].items():
    m["wall_ms_best"] = min(m["wall_ms"])
    m["gemm_ms_best"] = min(m["gemm_ms"])
out["speedup_wall"] = out["modes"]["0"]["wall_ms_best"] / out["modes"]["1"]["wall_ms_best"]
out["speedup_gemm"] = out["modes"]["0"]["gemm_ms_best"] / out["modes"]["1"]["gemm_ms_best"]
print(json.dumps(out))
