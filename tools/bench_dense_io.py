"""Ingest and egress of a whole dense matrix (MatfastSession.fromDense, Dataset.toTorch / toNumpy, mr_matrix_to_dense) at N = 16384,
blk 1024, one JSON line per case.

Cases, in both directions: device <-> device with the matrix row-major and column-major (the blocks keep its layout: line copies),
a layout change (column-major blocks assembled into a row-major tensor: the shared-memory transpose), and pinned and pageable host
memory.  Each time is the median of CUDA-event intervals on torch's current stream over repeated calls after warm-up (an ingest is
closed by ordering that stream behind the ingest stream).  GB/s counts the compulsory bytes, 2 N^2 8 (every element read once and
written once).  Device cases are set against the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s -- a data-sheet figure, not a
measurement; host cases against the same bytes moved by one plain torch copy in the same direction, timed the same way.  The card's
name, power limit and maximum SM clock are read in the same run.

    python tools/bench_dense_io.py [--n 16384] [--blk 1024] [--reps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_DATASHEET_BPS = 3.35e12


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip() if r.returncode == 0 else "unknown (nvidia-smi failed)"


def timed(fn, reps: int, warmup: int) -> float:
    """Median seconds of fn() between two events on torch's current stream."""
    cur = torch.cuda.current_stream()
    times = []
    for k in range(warmup + reps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record(cur)
        fn()
        end.record(cur)
        end.synchronize()
        if k >= warmup:
            times.append(start.elapsed_time(end) / 1e3)
    return statistics.median(times)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--blk", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dense_io needs a CUDA device")
    import matrel_b200 as mb
    from matrel_b200 import _native as N
    from matrel_b200.dataset import _torch_stream

    n, blk = a.n, a.blk
    card = gpu_info()
    compulsory = 2 * n * n * 8
    dev = torch.device("cuda", 0)
    cur = lambda: _torch_stream(dev)  # noqa: E731

    def report(direction, case, t, baseline=None, baseline_s=None):
        rec = {"direction": direction, "case": case, "n": n, "blk": blk, "median_s": round(t, 6),
               "gb_per_s": round(compulsory / t / 1e9, 1)}
        if baseline is None:
            rec["share_of_datasheet_hbm"] = round(compulsory / HBM_DATASHEET_BPS / t, 3)
        else:
            rec["plain_copy"] = baseline
            rec["plain_copy_s"] = round(baseline_s, 6)
            rec["vs_plain_copy"] = round(baseline_s / t, 3)
        rec["gpu"] = card
        print(json.dumps(rec), flush=True)

    torch.manual_seed(0)
    rm_dev = torch.rand(n, n, dtype=torch.float64, device=dev)              # row-major
    cm_dev = torch.rand(n, n, dtype=torch.float64, device=dev).t()          # column-major view
    pinned = torch.rand(n, n, dtype=torch.float64).pin_memory()
    pageable = np.random.default_rng(0).uniform(0, 1, (n, n))

    with mb.MatfastSession(device=0) as s:
        def ingest(src):
            def fn():
                ds = s.fromDense(src, blk)
                s.wait_ingest_on(cur())  # the current stream (and its end event) behind the ingest stream
                return ds
            return fn

        def to_device(ds, out, row_major):
            ld = out.stride(0) if row_major else out.stride(1)
            N.check(N.lib.mr_matrix_to_dense(ds._h, n, n, blk, C.c_void_p(out.data_ptr()), ld, row_major, C.c_void_p(cur())))
            return out

        report("ingest", "device_rowmajor", timed(ingest(rm_dev), a.reps, a.warmup))
        report("ingest", "device_colmajor", timed(ingest(cm_dev), a.reps, a.warmup))
        dev_buf = torch.empty(n, n, dtype=torch.float64, device=dev)
        t_h2d_pin = timed(lambda: dev_buf.copy_(pinned, non_blocking=True), a.reps, a.warmup)
        report("ingest", "pinned_host", timed(ingest(pinned), a.reps, a.warmup), "torch copy pinned -> device", t_h2d_pin)
        pageable_t = torch.from_numpy(pageable)
        t_h2d_page = timed(lambda: dev_buf.copy_(pageable_t), a.reps, a.warmup)
        report("ingest", "pageable_host", timed(ingest(pageable), a.reps, a.warmup), "torch copy pageable -> device", t_h2d_page)
        del dev_buf

        ds_rm, ds_cm = s.fromDense(rm_dev, blk), s.fromDense(cm_dev, blk)
        s.sync()
        out_rm = torch.empty(n, n, dtype=torch.float64, device=dev)
        out_cm = torch.empty(n, n, dtype=torch.float64, device=dev).t()
        report("egress", "device_rowmajor", timed(lambda: to_device(ds_rm, out_rm, 1), a.reps, a.warmup))
        ok = torch.equal(out_rm, rm_dev)
        report("egress", "device_colmajor", timed(lambda: to_device(ds_cm, out_cm, 0), a.reps, a.warmup))
        ok = ok and torch.equal(out_cm, cm_dev)
        report("egress", "device_layout_change", timed(lambda: to_device(ds_cm, out_rm, 1), a.reps, a.warmup))
        ok = ok and torch.equal(out_rm, cm_dev)
        del out_cm
        out_pin = torch.empty(n, n, dtype=torch.float64).pin_memory()
        t_d2h_pin = timed(lambda: out_pin.copy_(rm_dev, non_blocking=True), a.reps, a.warmup)

        def to_pinned():
            N.check(N.lib.mr_matrix_to_dense(ds_rm._h, n, n, blk, C.c_void_p(out_pin.data_ptr()), n, 1, C.c_void_p(cur())))
        report("egress", "pinned_host", timed(to_pinned, a.reps, a.warmup), "torch copy device -> pinned", t_d2h_pin)
        ok = ok and torch.equal(out_pin, rm_dev.cpu())
        out_page = torch.empty(n, n, dtype=torch.float64)
        t_d2h_page = timed(lambda: out_page.copy_(rm_dev), a.reps, a.warmup)
        got = np.zeros((n, n))

        def to_pageable():
            N.check(N.lib.mr_matrix_to_dense(ds_rm._h, n, n, blk, C.c_void_p(got.ctypes.data), n, 1, None))
        report("egress", "pageable_host", timed(to_pageable, a.reps, a.warmup), "torch copy device -> pageable", t_d2h_page)
        ok = ok and np.array_equal(got, out_page.numpy())
        # toNumpy as a user calls it: the array is new every time, so its pages are first touched by the copy
        t_new = timed(lambda: torch.empty(n, n, dtype=torch.float64).copy_(rm_dev), a.reps, a.warmup)
        report("egress", "pageable_host_new_array", timed(lambda: ds_rm.toNumpy(n, n, blk), a.reps, a.warmup),
               "torch copy device -> new pageable tensor", t_new)
    print(json.dumps({"summary": "dense_io", "n": n, "blk": blk, "exact": bool(ok), "gpu": card}), flush=True)
    if not ok:
        sys.exit("an egress did not reproduce its source exactly")


if __name__ == "__main__":
    main()
