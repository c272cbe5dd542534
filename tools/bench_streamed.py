"""The streamed multiply on one GPU: host-resident operands larger than device memory, and its cost against the resident product.

    python tools/bench_streamed.py [OUT_DIR] [--reps 3] [--n 65536] [--blk 2048] [--pair-n 32768]

1. N = 65536 (blk 2048), A, B and C host-resident (96 GiB of page-locked host memory).  When /proc/meminfo's MemAvailable is
   short of that, N = 49152 instead, and the output says so.  A and B come from mr_matrix_rand on the device (the benchmark's
   java.util.Random streams) and are moved to the host one at a time, so nothing this size passes through numpy.  One warm-up,
   then the median wall time of --reps calls (host clock around the call plus mr_sync), fp64-equivalent TFLOP/s (2 N^3 / t),
   tiles, h2d / d2h bytes and the effective PCIe rate.  Checks: Freivalds (C x = A (B x) over every block, the mat-vecs on the
   exact kernel) and numpy fp64 on a seeded sample of blocks.
2. N = 32768: the resident and the streamed product alternate in the same process, the streamed one under a stream_budget_mb that
   gives at least 4 tiles.  Reports the overhead of streaming and asserts that the two results are bit-identical.

One JSON line per run goes to stdout and OUT_DIR/bench_streamed.jsonl, with the GPU name, power limit and max SM clock read in
the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import matrel_b200 as mb  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0].strip() if r.returncode == 0 else "unknown"


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def host_rand(s, n, blk, seed):
    d = s.rand(n, n, blk, seed)
    h = d.toHost()
    s.sync()
    del d
    return h


def vector(s, x, blk):
    n = x.size
    return s.createDataset(mb.MatrixBlock(i, 0, mb.DenseMatrix(min(blk, n - i * blk), 1, x[i * blk:(i + 1) * blk].copy()))
                           for i in range(-(-n // blk)))


def collect_vector(ds, n, blk):
    out = np.zeros(n)
    for b in ds.collect():
        out[b.rid * blk:b.rid * blk + b.matrix.numRows] = b.matrix.to_numpy()[:, 0]
    return out


def freivalds(s, A, B, C, n, blk, rng):
    """max over rows of |C x - A (B x)| / (|A (B x)| + n 1e-3), every product on the exact kernel."""
    s.set_option("gemm_algo", 1)
    x = rng.uniform(-1, 1, n)
    dx = vector(s, x, blk)
    ABx = collect_vector(A.matrixMultiply(n, n, B.matrixMultiply(n, n, dx, n, 1, blk), n, 1, blk), n, blk)
    Cx = collect_vector(C.matrixMultiply(n, n, dx, n, 1, blk), n, blk)
    s.set_option("gemm_algo", 0)
    return float(np.max(np.abs(Cx - ABx) / (np.abs(ABx) + n * 1e-3)))


def sample_check(A, B, C, n, blk, rng, count):
    """max relative error of sampled C blocks against numpy fp64 (relative to |A| |B| of the block)."""
    nb = n // blk
    worst = 0.0
    for _ in range(count):
        i, j = (int(v) for v in rng.integers(0, nb, 2))
        a = np.hstack([A.get_block(i, k).to_numpy() for k in range(nb)])
        b = np.vstack([B.get_block(k, j).to_numpy() for k in range(nb)])
        ref, mag = a @ b, np.abs(a) @ np.abs(b)
        worst = max(worst, float(np.max(np.abs(C.get_block(i, j).to_numpy() - ref) / mag)))
    return worst


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(os.path.join(out, "bench_streamed.jsonl"), "a") as f:
            f.write(line + "\n")


def large_run(args, info, out):
    n, blk = args.n, args.blk
    note = None
    need = 3 * n * n * 8 + (8 << 30)
    if mem_available() < need:
        note = f"MemAvailable {mem_available() >> 30} GiB < {need >> 30} GiB needed at N = {n}: running N = 49152 instead"
        n = 49152
    rng = np.random.default_rng(n)
    with mb.MatfastSession(device=0) as s:
        A, B = host_rand(s, n, blk, 42), host_rand(s, n, blk, 43)
        C = A.matrixMultiply(n, n, B, n, n, blk)  # warm-up (also pins the result's host memory once)
        s.sync()
        del C
        times = []
        for _ in range(args.reps):
            s.reset_stats()
            t0 = time.perf_counter()
            C = A.matrixMultiply(n, n, B, n, n, blk)
            s.sync()
            times.append(time.perf_counter() - t0)
            st = s.stats()
            if len(times) < args.reps:
                del C
        t = statistics.median(times)
        rec = {"run": "streamed", "N": n, "blk": blk, "reps": args.reps, "median_s": round(t, 3),
               "spread": round((max(times) - min(times)) / t, 3), "tflops_fp64_equiv": round(2 * n ** 3 / t / 1e12, 2),
               "stream_tiles": st["stream_tiles"], "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
               "operand_h2d_bytes": st["stream_h2d_bytes"], "result_d2h_bytes": st["stream_d2h_bytes"],
               "pcie_gb_s": round((st["h2d_bytes"] + st["d2h_bytes"]) / t / 1e9, 1), "gpu": info}
        if note:
            rec["note"] = note
        rec["freivalds_max_rel"] = freivalds(s, A, B, C, n, blk, rng)
        rec["numpy_sample_max_rel"] = sample_check(A, B, C, n, blk, rng, 2)
        rec["checks_pass"] = rec["freivalds_max_rel"] <= 1e-11 and rec["numpy_sample_max_rel"] <= 1e-12
        emit(out, rec)
        del A, B, C  # datasets go before their session: the page-locked memory is handed back


def pair_run(args, info, out):
    n, blk = args.pair_n, args.blk
    with mb.MatfastSession(device=0) as s:
        A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
        hA, hB = A.toHost(), B.toHost()
        budget = None
        for gib in (24, 16, 12, 8, 6, 4):  # the largest budget that still cuts C into at least 4 tiles
            s.set_option("stream_budget_mb", gib << 10)
            s.reset_stats()
            try:
                C = hA.matrixMultiply(n, n, hB, n, n, blk)
            except MemoryError:
                continue
            s.sync()
            del C
            if s.stats()["stream_tiles"] >= 4:
                budget = gib << 10
                break
        assert budget is not None, "no budget gives 4 tiles"
        s.set_option("stream_budget_mb", budget)
        R = A.matrixMultiply(n, n, B, n, n, blk)
        s.sync()
        del R
        tr, ts = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            R = A.matrixMultiply(n, n, B, n, n, blk)
            s.sync()
            tr.append(time.perf_counter() - t0)
            s.reset_stats()
            t0 = time.perf_counter()
            C = hA.matrixMultiply(n, n, hB, n, n, blk)
            s.sync()
            ts.append(time.perf_counter() - t0)
            tiles = s.stats()["stream_tiles"]
            identical = all(np.array_equal(C.get_block(i, j).values.view(np.int64), R.get_block(i, j).values.view(np.int64))
                            for i, j in R.block_ids()) and sorted(C.block_ids()) == sorted(R.block_ids())
            assert identical, "streamed and resident products differ"
            del R, C
        del A, B, hA, hB
        r, t = statistics.median(tr), statistics.median(ts)
        emit(out, {"run": "resident_vs_streamed", "N": n, "blk": blk, "reps": args.reps, "stream_budget_mb": budget,
                   "stream_tiles": tiles, "resident_median_s": round(r, 3), "streamed_median_s": round(t, 3),
                   "resident_tflops": round(2 * n ** 3 / r / 1e12, 2), "streamed_tflops": round(2 * n ** 3 / t / 1e12, 2),
                   "overhead": round(t / r - 1, 3), "bit_identical": True, "gpu": info})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--blk", type=int, default=2048)
    ap.add_argument("--pair-n", type=int, default=32768)
    args = ap.parse_args()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    info = gpu_info()
    pair_run(args, info, args.out)
    large_run(args, info, args.out)


if __name__ == "__main__":
    main()
