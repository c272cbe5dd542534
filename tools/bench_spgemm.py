"""Sparse x sparse block products: `sprand` A x B with blk 1024 through the public API (so the same script measures any build).

Workloads (--workloads, comma separated): 32768:1e-3 (the chains end sparse), 32768:1.3e-2 (they end dense; the device sprand
draws at most ~14000 entries per 1024 x 1024 block, so 2e-2 is out of its reach), 65536:1e-3 (needs the native sparse product:
its dense images would take 96 GiB).  Per workload, one JSON line: the median and spread of the wall time of
one multiply (host-synchronised, after a warm-up), the scalar products and nnz(C) counted on the host from the blocks' structure,
products per second, the compulsory bytes 12 (nnz A + nnz B + nnz C) over the time against the 3.35 TB/s H100 SXM data-sheet
figure, and the GPU's name, power limit and maximum SM clock read in the same run.  --dump DIR writes four sampled output blocks
(dense m x n arrays) per workload, to compare two builds.

    python tools/bench_spgemm.py [--workloads 32768:1e-3,32768:1.3e-2] [--reps 5] [--warmup 1] [--dump DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import matrel_b200 as mb  # noqa: E402
from matrel_b200.dataset import sprand  # noqa: E402

HBM_TBPS = 3.35  # H100 SXM data-sheet HBM3 bandwidth


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def structure(ds, nb):
    """{(i, j): (nnz per column, nnz per row, nnz)} of a sparse dataset."""
    out = {}
    for i in range(nb):
        for j in range(nb):
            m = ds.get_block(i, j)
            lines = np.diff(m.colPtrs).astype(np.int64)
            per_minor = np.bincount(m.rowIndices, minlength=m.numRows if not m.isTransposed else m.numCols).astype(np.int64)
            cols, rows = (per_minor, lines) if m.isTransposed else (lines, per_minor)
            out[(i, j)] = (cols, rows, int(m.values.size))
    return out


def nnz_of(m) -> int:
    return int(m.values.size) if isinstance(m, mb.SparseMatrix) else int(np.count_nonzero(m.values))


def dense_of(m) -> np.ndarray:
    return m.to_numpy()


def run(s, n, density, reps, warmup, dump):
    blk = 1024
    nb = n // blk
    A = sprand(s, n, n, blk, density, 11, csr=True)
    B = sprand(s, n, n, blk, density, 12, csr=True)
    s.sync()
    sa, sb = structure(A, nb), structure(B, nb)
    products = 0
    for k in range(nb):
        ca = sum(sa[(i, k)][0] for i in range(nb))
        rb = sum(sb[(k, j)][1] for j in range(nb))
        products += int(np.dot(ca, rb))
    nnz_a = sum(v[2] for v in sa.values())
    nnz_b = sum(v[2] for v in sb.values())
    times = []
    C = None
    for r in range(warmup + reps):
        C = None
        s.sync()
        t0 = time.perf_counter()
        C = A.matrixMultiply(n, n, B, n, n, blk)
        s.sync()
        if r >= warmup:
            times.append(time.perf_counter() - t0)
    st = s.stats()
    nnz_c, kinds = 0, {}
    for i in range(nb):
        for j in range(nb):
            m = C.get_block(i, j)
            nnz_c += nnz_of(m)
            k = "dense" if isinstance(m, mb.DenseMatrix) else ("csr" if m.isTransposed else "csc")
            kinds[k] = kinds.get(k, 0) + 1
    if dump:
        os.makedirs(dump, exist_ok=True)
        picks = [(0, 0), (nb - 1, nb - 1), (3, nb // 2), (nb // 2, 5)]
        np.savez(os.path.join(dump, f"C_{n}_{density:g}.npz"), **{f"b{i}_{j}": dense_of(C.get_block(i, j)) for i, j in picks})
    med = float(np.median(times))
    byts = 12 * (nnz_a + nnz_b + nnz_c)
    return {"workload": f"sprand A x B, N={n}, blk={blk}, density={density:g}", "median_s": round(med, 4),
            "min_s": round(min(times), 4), "max_s": round(max(times), 4), "reps": reps,
            "scalar_products": products, "kernel_products": int(st.get("spgemm_products", -1)) if "spgemm_products" in st else None,
            "nnz_a": nnz_a, "nnz_b": nnz_b, "nnz_c": nnz_c, "output_formats": kinds,
            "products_per_s": round(products / med, 1),
            "compulsory_bytes": byts, "compulsory_tb_per_s": round(byts / med / 1e12, 4),
            "fraction_of_3.35TBps_datasheet": round(byts / med / 1e12 / HBM_TBPS, 5), "gpu": gpu_info()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="32768:1e-3,32768:1.3e-2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dump", default="")
    a = ap.parse_args()
    with mb.MatfastSession(device=0) as s:
        for w in a.workloads.split(","):
            n, d = w.split(":")
            print(json.dumps(run(s, int(n), float(d), a.reps, a.warmup, a.dump)), flush=True)


if __name__ == "__main__":
    main()
