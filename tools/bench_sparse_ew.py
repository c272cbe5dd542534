"""Element-wise joins of low-density sparse datasets (addElement / multiplyElement / divideElement on `sprand` pairs) through the
public API, on the stored-entry kernels (DESIGN section 4.5.3).

Workloads: N in {32768, 65536, 131072} x density {1e-4, 1e-3, 1e-2} x {CSR, CSC} for add and multiply, and divide at N = 16384
(its result is dense NaN wherever neither operand stores an entry), blk 1024.  The engine runs on the process's torch stream and
CUDA events bracket each whole call, host synchronisation included; median and range of --reps timed calls after --warmup.
Compulsory bytes: 12 bytes per stored entry of A, B and a sparse C (value and row index), 4 per column pointer, 8 per element of
a dense C; over the median time, against the 3.35 TB/s H100 SXM data-sheet figure.  One JSON line per workload, with the GPU's
name and power limit read in the same run.

With --digest each record also carries a SHA-256 over the result's blocks (ids, kind, column pointers, row indices and value bits,
NaNs canonicalised), so that runs of two builds can be compared.

    python tools/bench_sparse_ew.py [--workloads add:32768:1e-3:csr,...] [--reps 5] [--warmup 1] [--digest]
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import matrel_b200 as mb  # noqa: E402
from matrel_b200 import _native as N  # noqa: E402
from matrel_b200.dataset import sprand  # noqa: E402

HBM_TBPS = 3.35  # H100 SXM data-sheet HBM3 bandwidth
BLK = 1024
FN = {"add": "addElement", "mul": "multiplyElement", "div": "divideElement"}


def default_workloads():
    w = [f"{op}:{n}:{d}:{f}" for n in (32768, 65536, 131072) for d in ("1e-4", "1e-3", "1e-2") for f in ("csr", "csc")
         for op in ("add", "mul")]
    return w + [f"div:16384:{d}:{f}" for d in ("1e-4", "1e-3", "1e-2") for f in ("csr", "csc")]


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def stored_bytes(ds) -> tuple:
    """(compulsory bytes of the dataset's blocks, stored entries of its sparse blocks), from block sizes only."""
    total, nnz = 0, 0
    for rid, cid in ds.block_ids():
        d = N.mr_block_desc()
        N.check(N.lib.mr_matrix_get_block(ds._h, rid, cid, C.byref(d)))
        if d.type == 0:
            total += 12 * d.valuesLen + 4 * d.colPtrsLen
            nnz += d.valuesLen
        else:
            total += 8 * d.valuesLen
    return total, nnz


def digest(ds) -> str:
    import numpy as np
    h = hashlib.sha256()
    for rid, cid in ds.block_ids():
        m = ds.get_block(rid, cid)
        v = np.array(m.values, dtype=np.float64)
        v[np.isnan(v)] = np.nan
        h.update(repr((rid, cid, type(m).__name__, m.numRows, m.numCols, bool(m.isTransposed))).encode())
        if type(m).__name__ == "SparseMatrix":
            h.update(np.asarray(m.colPtrs, np.int32).tobytes())
            h.update(np.asarray(m.rowIndices, np.int32).tobytes())
        h.update(v.tobytes())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(default_workloads()))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--digest", action="store_true")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    gpu = gpu_info()
    stream = torch.cuda.current_stream()
    s = mb.MatfastSession(device=0, stream=stream.cuda_stream)
    for w in args.workloads.split(","):
        op, n, dens, fmt = w.split(":")
        n, dens = int(n), float(dens)
        A = sprand(s, n, n, BLK, dens, 1, csr=(fmt == "csr"))
        B = sprand(s, n, n, BLK, dens, 2, csr=(fmt == "csr"))
        fn = getattr(A, FN[op])
        for _ in range(args.warmup):
            fn(n, n, B, n, n, BLK)
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            Cds = fn(n, n, B, n, n, BLK)
            e1.record(stream)
            e1.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
            del Cds
        s.reset_stats()
        Cds = fn(n, n, B, n, n, BLK)
        st = s.stats()
        (ba, na), (bb, nb), (bc, nc) = stored_bytes(A), stored_bytes(B), stored_bytes(Cds)
        times.sort()
        med = times[len(times) // 2]
        rec = {"workload": w, "op": op, "n": n, "density": dens, "format": fmt, "blk": BLK, "median_s": med,
               "min_s": times[0], "max_s": times[-1], "nnz_a": na, "nnz_b": nb, "nnz_c": nc,
               "ew_sparse_pairs": st.get("ew_sparse_pairs"), "ew_sparse_entries": st.get("ew_sparse_entries"),
               "kernel_launches": st["kernel_launches"], "compulsory_bytes": ba + bb + bc,
               "bytes_per_s": (ba + bb + bc) / med, "share_of_3_35_TBps": (ba + bb + bc) / med / (HBM_TBPS * 1e12),
               "gpu": gpu}
        if args.digest:
            rec["digest"] = digest(Cds)
        print(json.dumps(rec), flush=True)
        del A, B, Cds
        s.sync()
    s.stop()


if __name__ == "__main__":
    main()
