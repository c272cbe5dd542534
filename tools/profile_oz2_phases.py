"""Per-kernel split of one Ozaki-II fp64 multiply (the bench workload by default): python tools/profile_oz2_phases.py [N] [BLK] [OUT_DIR]
[key=value ...] -> one JSON line with the device time of every kernel name over one multiply (absmax, exponents, residues, int8 GEMM,
CRT, fixup, ...), the sum, and the host-timed multiply without the profiler.  key=value pairs are session options (for example
oz2_strassen=0).  The torch.profiler trace is written under OUT_DIR (default: oz2_profile in the temporary directory)."""
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import matrel_b200 as mb  # noqa: E402

pos = [a for a in sys.argv[1:] if "=" not in a]
opts = dict(a.split("=", 1) for a in sys.argv[1:] if "=" in a)
n = int(pos[0]) if len(pos) > 0 else 16384
blk = int(pos[1]) if len(pos) > 1 else 1024
out_dir = pos[2] if len(pos) > 2 else os.path.join(tempfile.gettempdir(), "oz2_profile")
os.makedirs(out_dir, exist_ok=True)

with mb.MatfastSession(device=0) as s:
    for k, v in opts.items():
        s.set_option(k, int(v))
    A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
    for _ in range(2):
        C = A.matrixMultiply(n, n, B, n, n, blk)
        del C
    s.sync()
    reps = 3
    t0 = time.perf_counter()
    for _ in range(reps):
        C = A.matrixMultiply(n, n, B, n, n, blk)
        del C
    s.sync()
    wall = (time.perf_counter() - t0) / reps * 1e3
    s.reset_stats()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        C = A.matrixMultiply(n, n, B, n, n, blk)
        s.sync()
    st = s.stats()
    del C
    prof.export_chrome_trace(os.path.join(out_dir, "oz2_multiply.pt.trace.json"))

kernels = {}
for ev in prof.key_averages():
    dev_us = getattr(ev, "device_time_total", None)
    if dev_us is None:
        dev_us = getattr(ev, "cuda_time_total", 0)
    if dev_us <= 0:
        continue
    kernels[ev.key[:90]] = {"ms": round(dev_us / 1e3, 3), "calls": int(ev.count)}
total = sum(v["ms"] for v in kernels.values())
out = {"n": n, "blk": blk, "options": opts, "wall_ms_unprofiled": round(wall, 3), "device_ms_sum": round(total, 3),
       "kernels": dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms"])),
       "stats": {k: st[k] for k in ("tc_int8_ops", "tc_moduli", "tc_strassen_jobs") if k in st},
       "gpu": torch.cuda.get_device_name(0)}
print(json.dumps(out))
