"""A/B of the two Ozaki-II int8 GEMM kernels on ONE box, back to back: the CTA-pair kernel (ozaki2_gemm_2sm_kernel, gemm_variant 0)
against the single-CTA kernel (ozaki_gemm_i8_kernel, gemm_variant 2).  python tools/ab_paired.py [N] [BLK] [REPS] -> one JSON line
with the whole-multiply wall time (context synchronised) and the int8 GEMM launch time (events inside the library) per kernel,
interleaved 0 / 2 / 0 / 2 so that clock drift under the power cap hits both alike, plus a bit-identity check of one output block."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import matrel_b200 as mb

n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
blk = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 4
names = {0: "pair", 2: "single"}
out = {"n": n, "blk": blk, "reps": reps, "kernels": {}}
with mb.MatfastSession(device=0) as s:
    s.set_option("gemm_algo", 0)
    A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
    ref = {}
    for rnd in range(2):
        for variant in (0, 2):
            s.set_option("gemm_variant", variant)
            s.set_option("time_kernels", 0)
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
            for _ in range(2):
                C = A.matrixMultiply(n, n, B, n, n, blk)
            st = s.stats()
            ref.setdefault(variant, C.get_block(1, 2).values.copy())
            del C
            m = out["kernels"].setdefault(names[variant], {"wall_ms": [], "gemm_ms": []})
            m["wall_ms"].append(round(wall, 3))
            m["gemm_ms"].append(round(st["tc_gemm_ms_total"] / 2, 3))
            m["moduli"] = int(st.get("tc_moduli", 0))
    s.set_option("gemm_variant", -1)
    out["bit_identical_block"] = bool(np.array_equal(ref[0], ref[2]))
for m in out["kernels"].values():
    m["wall_ms_best"] = min(m["wall_ms"])
    m["gemm_ms_best"] = min(m["gemm_ms"])
out["single_over_pair_gemm"] = out["kernels"]["single"]["gemm_ms_best"] / out["kernels"]["pair"]["gemm_ms_best"]
print(json.dumps(out))
