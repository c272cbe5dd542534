"""C-stationary (mr_dmatrix_multiply) against K-split (mr_dmatrix_multiply_ksplit) on the single-process grid of every visible GPU.

    python tools/bench_grid_ksplit.py OUT_DIR [--reps 10] [--warmup 2] [--gemm-algo 0] [--shapes gram,wtw,wtv,square]

Shapes (blk 1024): the Gram matrix X^T X with X = 262144 x 2048, W^T W with W = 65536 x 1024, W^T V with V = 65536 x 16384 (the
transposed operand comes from mr_dmatrix_transpose, as a user writes it), and the N = 16384 square product for comparison.  The two
modes run alternately in the same process after a warm-up; every repetition is a host clock around the call plus mr_grid_sync.
One JSON line per shape and mode goes to OUT_DIR/bench_grid_ksplit.jsonl (and stdout): median and spread of the time,
fp64-equivalent TFLOP/s (2 M N K / t), p2p_bytes of one call, the max relative difference between the two modes and against numpy
fp64 on sampled C blocks, and the GPU name / power limit / max SM clock read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from matrel_b200 import _native as N  # noqa: E402

SHAPES = {  # name: (rows of the stored left operand, its cols, cols of the right operand, transposed left operand)
    "gram": (262144, 2048, 2048, True),     # X^T X
    "wtw": (65536, 1024, 1024, True),       # W^T W
    "wtv": (65536, 1024, 16384, True),      # W^T V
    "square": (16384, 16384, 16384, False),  # A B, BASELINE configs[2]
}
BLK = 1024


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"nvidia-smi failed: {r.stderr.strip()}")
    return [line.strip() for line in r.stdout.strip().splitlines()[1:]]


def p2p(g, n):
    total = 0
    for r in range(n):
        ctx, st = C.c_void_p(), N.mr_stats()
        N.check(N.lib.mr_grid_context(g, r, C.byref(ctx)))
        N.check(N.lib.mr_get_stats(ctx, C.byref(st)))
        total += st.p2p_bytes
    return total


def block(dm, rid, cid):
    """Block (rid, cid) as a 2-D numpy array, whatever its layout flag."""
    d = N.mr_block_desc()
    N.check(N.lib.mr_dmatrix_get_block(dm, rid, cid, C.byref(d)))
    v = np.empty(d.valuesLen)
    d.values = v.ctypes.data_as(C.POINTER(C.c_double))
    N.check(N.lib.mr_dmatrix_get_block(dm, rid, cid, C.byref(d)))
    return v.reshape(d.numRows, d.numCols) if d.isTransposed else v.reshape(d.numCols, d.numRows).T


def run_shape(g, n, name, args, info):
    rows, cols, ncols_b, transposed = SHAPES[name]
    handles = []
    if transposed:   # A = X^T (flag-transposed slabs), B = X or V
        X, A = C.c_void_p(), C.c_void_p()
        N.check(N.lib.mr_dmatrix_rand(g, rows, cols, BLK, 101, C.byref(X)))
        N.check(N.lib.mr_dmatrix_transpose(X, C.byref(A)))
        if ncols_b == cols:
            B = X
        else:
            B = C.c_void_p()
            N.check(N.lib.mr_dmatrix_rand(g, rows, ncols_b, BLK, 202, C.byref(B)))
            handles.append(B)
        handles += [X, A]
        M, K, Ncol = cols, rows, ncols_b
    else:
        A, B = C.c_void_p(), C.c_void_p()
        N.check(N.lib.mr_dmatrix_rand(g, rows, cols, BLK, 101, C.byref(A)))
        N.check(N.lib.mr_dmatrix_rand(g, cols, ncols_b, BLK, 202, C.byref(B)))
        handles += [A, B]
        M, K, Ncol = rows, cols, ncols_b
    N.check(N.lib.mr_grid_sync(g))
    modes = {"cstationary": N.lib.mr_dmatrix_multiply, "ksplit": N.lib.mr_dmatrix_multiply_ksplit}

    def call(mode):
        out = C.c_void_p()
        t0 = time.perf_counter()
        N.check(modes[mode](A, B, C.byref(out)))
        N.check(N.lib.mr_grid_sync(g))
        return time.perf_counter() - t0, out

    moved, results = {}, {}
    for mode in modes:  # warm-up; the first call of each mode also yields its p2p bytes and its result for the accuracy check
        for w in range(max(1, args.warmup)):
            before = p2p(g, n)
            _, out = call(mode)
            if w == 0:
                moved[mode] = p2p(g, n) - before
                results[mode] = out
            else:
                N.check(N.lib.mr_dmatrix_free(out))
    times = {m: [] for m in modes}
    order = list(modes)
    for rep in range(args.reps):
        for mode in (order if rep % 2 == 0 else order[::-1]):
            t, out = call(mode)
            times[mode].append(t)
            N.check(N.lib.mr_dmatrix_free(out))
    # accuracy on sampled C blocks: the two modes against each other and against numpy fp64 from the operand blocks
    nbi, nbj, nbk = -(-M // BLK), -(-Ncol // BLK), -(-K // BLK)
    rng = np.random.default_rng(5)
    samples = sorted({(int(rng.integers(nbi)), int(rng.integers(nbj))) for _ in range(2)})
    diff_modes = diff_ref = 0.0
    for (i, j) in samples:
        ref = sum(block(A, i, k) @ block(B, k, j) for k in range(nbk))
        cs, ks = block(results["cstationary"], i, j), block(results["ksplit"], i, j)
        scale = np.max(np.abs(ref))
        diff_modes = max(diff_modes, float(np.max(np.abs(ks - cs)) / scale))
        diff_ref = max(diff_ref, float(max(np.max(np.abs(ks - ref)), np.max(np.abs(cs - ref))) / scale))
    for out in results.values():
        N.check(N.lib.mr_dmatrix_free(out))
    for h in handles:
        N.check(N.lib.mr_dmatrix_free(h))
    lines = []
    for mode in modes:
        ts = sorted(times[mode])
        med = statistics.median(ts)
        lines.append({
            "tool": "bench_grid_ksplit", "shape": name, "mode": mode, "gpus": n, "M": M, "N": Ncol, "K": K, "blk": BLK,
            "gemm_algo": args.gemm_algo, "reps": len(ts), "median_s": med, "min_s": ts[0], "max_s": ts[-1],
            "spread": (ts[-1] - ts[0]) / med, "tflops_fp64_equiv": 2.0 * M * Ncol * K / med / 1e12, "p2p_bytes": moved[mode],
            "sampled_blocks": samples, "max_rel_diff_between_modes": diff_modes, "max_rel_diff_vs_numpy": diff_ref,
            "gpu": info,
        })
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gemm-algo", type=int, default=0)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    import torch
    n = torch.cuda.device_count()
    if n < 1:
        raise SystemExit("no GPU visible: this benchmark measures the grid on the device")
    info = gpu_info()
    os.makedirs(args.out_dir, exist_ok=True)
    g = C.c_void_p()
    N.check(N.lib.mr_init_grid(C.byref(N.mr_options(-1, 1, args.gemm_algo, 0, None)), n, C.byref(g)))
    try:
        with open(os.path.join(args.out_dir, "bench_grid_ksplit.jsonl"), "a") as f:
            for name in args.shapes.split(","):
                for line in run_shape(g, n, name, args, info):
                    print(json.dumps(line), flush=True)
                    f.write(json.dumps(line) + "\n")
    finally:
        N.check(N.lib.mr_grid_shutdown(g))


if __name__ == "__main__":
    main()
