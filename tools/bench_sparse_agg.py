"""Aggregates and slices of low-density sparse datasets (rowSum / colSum / trace / project / selection of `sprand` datasets) through
the public API, on the stored-entry kernels (DESIGN section 4.5.4).

Workloads: N in {32768, 65536, 131072} x density {1e-4, 1e-3, 1e-2} x {CSR, CSC}, blk 1024; with --dense, the same matrices stored
as dense blocks where they fit (N <= 65536), for comparison.  The engine runs on a torch stream of its own and CUDA events on it bracket
each whole call, host work included, followed by a synchronise; median and range of --reps timed calls after --warmup.
Compulsory bytes: 12 per stored entry read (value and index), 4 per line pointer, 8 per output element, and 8 per element an
operator reads of a dense block (all of them, a line, the diagonal or one entry); over the median time, against the 3.35 TB/s
H100 SXM data-sheet figure.  project / selection read only the blocks of one block row or column (one block); their bytes count
those blocks.  One JSON line per (workload, operator), with the GPU's
name, power limit and max SM clock read in the same run.

    python tools/bench_sparse_agg.py [--workloads 32768:1e-3:csr,...] [--reps 5] [--warmup 1] [--dense]
"""
from __future__ import annotations

import argparse
import ctypes as C
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


def default_workloads():
    return [f"{n}:{d}:{f}" for n in (32768, 65536, 131072) for d in ("1e-4", "1e-3", "1e-2") for f in ("csr", "csc")]


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def block_bytes(ds, keep=lambda rid, cid: True, dense_elems=None) -> tuple:
    """(compulsory bytes read from the kept blocks, their stored sparse entries), from block sizes only.  dense_elems: elements an
    operator reads of a dense block (a line, a diagonal, one entry), None = all of them."""
    total, nnz = 0, 0
    for rid, cid in ds.block_ids():
        if not keep(rid, cid):
            continue
        d = N.mr_block_desc()
        N.check(N.lib.mr_matrix_get_block(ds._h, rid, cid, C.byref(d)))
        if d.type == 0:
            total += 12 * d.valuesLen + 4 * d.colPtrsLen
            nnz += d.valuesLen
        else:
            total += 8 * (d.valuesLen if dense_elems is None else dense_elems)
    return total, nnz


def operators(n):
    """(name, call, which blocks it reads, elements it reads of a dense block (None = all), output elements)."""
    i, j = n // 3, (2 * n) // 3
    return [
        ("rowSum", lambda A: A.rowSum(n, n), lambda r, c: True, None, n),
        ("colSum", lambda A: A.colSum(n, n), lambda r, c: True, None, n),
        ("trace", lambda A: A.trace(n, n), lambda r, c: r == c, BLK, 1),
        ("project_row", lambda A: A.project(n, n, BLK, True, i), lambda r, c: r == i // BLK, BLK, n),
        ("project_col", lambda A: A.project(n, n, BLK, False, j), lambda r, c: c == j // BLK, BLK, n),
        ("selection", lambda A: A.selection(n, n, BLK, i, j), lambda r, c: (r, c) == (i // BLK, j // BLK), 1, 1),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(default_workloads()))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dense", action="store_true", help="also time the same matrices stored dense (N <= 65536)")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    gpu = gpu_info()
    stream = torch.cuda.Stream()  # a stream of its own: the engine's launches and the events are ordered on it
    s = mb.MatfastSession(device=0, stream=stream.cuda_stream)
    for w in args.workloads.split(","):
        n, dens, fmt = w.split(":")
        n, dens = int(n), float(dens)
        A = sprand(s, n, n, BLK, dens, 1, csr=(fmt == "csr"))
        kinds = [("sparse", A)]
        if args.dense and n <= 65536:
            kinds.append(("dense", A.materialize()))  # every block densified
        for kind, X in kinds:
            for name, call, keep, dense_elems, nout in operators(n):
                for _ in range(args.warmup):
                    call(X)
                times = []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    out = call(X)
                    e1.record(stream)
                    e1.synchronize()
                    times.append(e0.elapsed_time(e1) / 1e3)
                    del out
                s.reset_stats()
                out = call(X)
                s.sync()
                st = s.stats()
                del out
                nbytes, nnz = block_bytes(X, keep, dense_elems)
                nbytes += 8 * nout
                times.sort()
                med = times[len(times) // 2]
                rec = {"workload": w, "storage": kind, "op": name, "n": n, "density": dens, "format": fmt, "blk": BLK,
                       "median_s": med, "min_s": times[0], "max_s": times[-1], "nnz_read": nnz,
                       "agg_sparse_blocks": st["agg_sparse_blocks"], "agg_sparse_entries": st["agg_sparse_entries"],
                       "kernel_launches": st["kernel_launches"], "compulsory_bytes": nbytes, "bytes_per_s": nbytes / med,
                       "share_of_3_35_TBps": nbytes / med / (HBM_TBPS * 1e12), "gpu": gpu}
                print(json.dumps(rec), flush=True)
            if kind == "dense":
                del X
        del A, kinds
        s.sync()
    s.stop()


if __name__ == "__main__":
    main()
