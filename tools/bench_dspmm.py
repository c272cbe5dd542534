"""Dense x low-density sparse products A S through the public API, so that the same script measures any build.

The sparse side takes the stored-entry route (DESIGN section 4.5.2) where its density allows; the comparison is the same product
with S's blocks stored dense, which is what the densified route computes, run alternately in the same process.  Workloads
(--workloads, comma separated, N:density[:kind]):
  * 16384:1e-3, 16384:3e-3, 16384:1e-2 -- A a dense 16384^2 `rand`, S `sprand` (CSC);
  * 16384:2e-2:mask, 16384:3e-2:mask, 16384:1e-1:mask -- S from a masked dense matrix (beyond the ~1.3e-2 per 1024^2 block
    sprand reaches).  Above kDspmmMaxDensity both sides run the densified route (dspmm_pairs = 0); to find the crossover, build
    with the threshold at its cap of 0.1;
  * 65536:1e-3:wtv -- W^T V, W 65536 x 1024 `rand` (W^T flag-transposed), V sprand 65536^2 (its dense images take 32 GiB);
  * 131072:1e-4:wtv:only -- the same at N = 131072, the route only (the densified product needs 128 GiB).
Per workload one JSON line: median and spread of the host-synchronised time per multiply for each route, 2 dspmm_products per
second, compulsory bytes (A + 12 nnz + C) over the time against the 3.35 TB/s H100 SXM data sheet, the largest difference between
the two products relative to the largest |C|, and the GPU's name, power limit and maximum SM clock read in the same run.

    python tools/bench_dspmm.py [--workloads 16384:1e-3,...] [--reps 5] [--warmup 1]
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
BLK = 1024
DEFAULT = ("16384:1e-3,16384:3e-3,16384:1e-2,16384:2e-2:mask,16384:3e-2:mask,16384:1e-1:mask,65536:1e-3:wtv,"
           "131072:1e-4:wtv:only")


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def masked_sparse(s, n, density, seed):
    """n x n CSC blocks of U(0, 1) values kept with probability `density` (host-built)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n // BLK):
        for j in range(n // BLK):
            m = sp.random(BLK, BLK, density=density, format="csc", random_state=rng, dtype=np.float64)
            m.sort_indices()
            rows.append(mb.MatrixBlock(i, j, mb.SparseMatrix(BLK, BLK, m.indptr.astype(np.int32), m.indices.astype(np.int32),
                                                             m.data, False)))
    return s.createDataset(rows)


def densified(s, S, n):
    """S with every block stored dense and column-major (S^T assembled row-major is S column-major)."""
    import torch
    t = S.transpose().toTorch(n, n, BLK)
    D = s.fromDense(t.t(), BLK)
    D.wait_ingest()
    del t
    torch.cuda.empty_cache()
    return D


def timed(s, fn, reps, warmup):
    for _ in range(warmup):
        fn()
        s.sync()
    ts = []
    for _ in range(reps):
        s.sync()
        t0 = time.perf_counter()
        C = fn()
        s.sync()
        ts.append(time.perf_counter() - t0)
        del C
    return ts


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=DEFAULT)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    info = gpu_info()
    with mb.MatfastSession(device=0) as s:
        for w in args.workloads.split(","):
            parts = w.split(":")
            n, d, kinds = int(parts[0]), float(parts[1]), set(parts[2:])
            wtv = "wtv" in kinds
            if wtv:
                W = s.rand(n, BLK, BLK, 3)
                A, (ar, ac) = W.transpose(), (BLK, n)
            else:
                A, (ar, ac) = s.rand(n, n, BLK, 1), (n, n)
            S = masked_sparse(s, n, d, 2) if "mask" in kinds else sprand(s, n, n, BLK, d, 2, csr=False)
            s.sync()
            run = lambda B: A.matrixMultiply(ar, ac, B, n, n, BLK)  # noqa: E731
            s.reset_stats()
            C = run(S)
            s.sync()
            st = s.stats()
            nnz = st["dspmm_products"] // ar if st["dspmm_pairs"] else None
            rec = {"workload": w, "rows": ar, "n": n, "density": d, "dspmm_pairs": st["dspmm_pairs"],
                   "dspmm_products": st["dspmm_products"]}
            route, dense_t = [], []
            D = None if "only" in kinds else densified(s, S, n)
            for _ in range(args.reps):  # alternate the two routes
                route += timed(s, lambda: run(S), 1, args.warmup if not route else 0)
                if D is not None:
                    dense_t += timed(s, lambda: run(D), 1, args.warmup if not dense_t else 0)
            med = float(np.median(route))
            rec["route_s"] = {"median": med, "min": float(min(route)), "max": float(max(route))}
            rec["flop_per_s"] = 2 * st["dspmm_products"] / med
            if nnz is not None:
                compulsory = 8 * ar * ac + 12 * nnz + 8 * ar * n
                rec["compulsory_bytes"] = compulsory
                rec["hbm_share"] = compulsory / med / (HBM_TBPS * 1e12)
            if D is not None:
                rec["densified_s"] = {"median": float(np.median(dense_t)), "min": float(min(dense_t)), "max": float(max(dense_t))}
                rec["speedup"] = float(np.median(dense_t)) / med
                import torch
                Cd = run(D)
                x, y = C.toTorch(ar, n, BLK), Cd.toTorch(ar, n, BLK)
                rec["max_rel_diff"] = float((x - y).abs().max() / y.abs().max().clamp_min(1e-300))
                del x, y, Cd, D
                torch.cuda.empty_cache()
            rec["gpu"] = info
            print(json.dumps(rec), flush=True)
            del C, S, A


if __name__ == "__main__":
    main()
