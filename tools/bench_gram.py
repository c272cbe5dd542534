"""Timing of Gram products (DESIGN section 4.1.2): C = A A^T and C = A^T A through the Gram route (A and A.t() share their arrays),
alternating in the same session with the general route on a copy of A (A.multiplyScalar(1.0): the same bits in other arrays).
Whole matrixMultiply calls are timed with CUDA events and a synchronise; median of --reps after a warm-up of each.  Every timed
shape asserts that both routes give identical bits.  One JSON line per case, with the card, its power limit and max SM clock.

  AAt:      A A^T, A 16384 x 16384, blk 1024 (the bench.py shape), auto engine (Ozaki-II)
  AtA:      A^T A, A 32768 x 16384, blk 1024, auto
  XtX:      X^T X, X 262144 x 2048, blk 1024: K >= 2^17, so DMMA computes 3 of the 4 blocks
  AAt_dmma: A A^T as AAt under gemm_algo 1

The mirror kernel's time comes from a separate torch.profiler run of one Gram call; its rate is the bytes it moves (every
strictly-lower element read once and written once) over that time, against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM
(a data-sheet number, not a measured one)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--cases", default="AAt,AtA,XtX,AAt_dmma")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import matrel_b200 as mb  # noqa: E402

BLK = 1024
DATASHEET_BPS = 3.35e12
CASES = {"AAt": ("AAt", 16384, 16384, 0), "AtA": ("AtA", 32768, 16384, 0), "XtX": ("AtA", 262144, 2048, 0),
         "AAt_dmma": ("AAt", 16384, 16384, 1)}
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()


def timed_call(s, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.sync()
    e0.record()
    out = fn()
    s.sync()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def mirror_ms(s, fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        s.sync()
        torch.cuda.synchronize()
    del out
    us = sum(e.device_time_total for e in prof.events() if "gram_mirror" in e.name)
    return us / 1e3 if us > 0 else None


def run_case(s, name):
    kind, m, n, algo = CASES[name]
    s.set_option("gemm_algo", algo)
    A = s.rand(m, n, BLK, 42)
    A2 = A.multiplyScalar(1.0)
    if kind == "AAt":
        N, gram, general = m, (lambda: A.matrixMultiply(m, n, A.t(), n, m, BLK)), (lambda: A.matrixMultiply(m, n, A2.t(), n, m, BLK))
    else:
        N, gram, general = n, (lambda: A.t().matrixMultiply(n, m, A, m, n, BLK)), (lambda: A2.t().matrixMultiply(n, m, A, m, n, BLK))
    for fn in (gram, general):   # warm-up
        fn()
    s.sync()
    s.reset_stats()
    Cg = gram()
    s.sync()
    st = s.stats()
    assert st["gram_blocks"] > 0, st
    Cr = general()
    s.sync()
    assert s.stats()["gram_blocks"] == 0
    same = np.array_equal(Cg.toNumpy(N, N, BLK).view(np.int64), Cr.toNumpy(N, N, BLK).view(np.int64))
    assert same, f"{name}: the Gram route differs from the general route"
    del Cg, Cr
    tg, tr = [], []
    for _ in range(args.reps):
        t, C = timed_call(s, gram)
        tg.append(t)
        del C
        t, C = timed_call(s, general)
        tr.append(t)
        del C
    mir = mirror_ms(s, gram)
    nb = -(-N // BLK)
    lower = N * (N - 1) // 2
    rec = {"case": name, "C": f"{N}x{N}", "K": m if kind == "AtA" else n, "blk": BLK, "gemm_algo": algo,
           "gram_ms": float(np.median(tg)), "general_ms": float(np.median(tr)), "speedup": float(np.median(tr) / np.median(tg)),
           "gram_blocks": st["gram_blocks"], "gram_mirrored_blocks": st["gram_mirrored_blocks"], "output_blocks": nb * nb,
           "tc_int8_ops": st["tc_int8_ops"], "same_bits": bool(same), "mirror_ms": mir,
           "mirror_TBps": (16 * lower / (mir * 1e-3) / 1e12) if mir else None,
           "mirror_of_datasheet_bw": (16 * lower / (mir * 1e-3) / DATASHEET_BPS) if mir else None,
           "gram_ms_all": tg, "general_ms_all": tr, "card": card}
    s.set_option("gemm_algo", 0)
    return rec


with mb.MatfastSession(device=0) as s:
    for name in args.cases.split(","):
        rec = run_case(s, name)
        line = json.dumps(rec)
        print(line, flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")
