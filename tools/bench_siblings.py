"""HBM-bound sibling operators at N x N fp64 (default 16384 / 1024-block): CUDA-event timings and
achieved GB/s against the algorithmic bytes of SURVEY.md section 8(d).
   python tools/bench_siblings.py [N] [BLK] [reps]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import matrel_b200 as mb

n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
blk = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
peak = 3350.0   # GB/s, H100 SXM data sheet (HBM3); a ceiling, not a measured rate
stream = torch.cuda.Stream()
with torch.cuda.stream(stream):
    s = mb.MatfastSession(device=0, stream=stream.cuda_stream)
    A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
    At = A.t()
    nn = n * n * 8
    cases = [
        ("addElement (N,N)", lambda: A.addElement(n, n, B, n, n, blk), 3 * nn),
        ("multiplyElement (N,N)", lambda: A.multiplyElement(n, n, B, n, n, blk), 3 * nn),
        ("divideElement (N,N)", lambda: A.divideElement(n, n, B, n, n, blk), 3 * nn),
        ("addElement (T,N) mixed layout", lambda: At.addElement(n, n, B, n, n, blk), 3 * nn),
        ("multiplyScalar", lambda: A.multiplyScalar(2.5), 2 * nn),
        ("addScalar", lambda: A.addScalar(2.5), 2 * nn),
        ("power(2.0)", lambda: A.power(2.0), 2 * nn),
        ("power(0.37)", lambda: A.power(0.37), 2 * nn),
        ("rowSum", lambda: A.rowSum(n, n), nn),
        ("colSum", lambda: A.colSum(n, n), nn),
        ("rowSum of transposed", lambda: At.rowSum(n, n), nn),
        ("sum", lambda: A.sum(n, n), nn),
        ("trace", lambda: A.trace(n, n), 0),
        ("project row", lambda: A.project(n, n, blk, True, n // 3), 0),
        ("transpose (flag only)", lambda: A.t(), 0),
        ("transpose + materialize", lambda: At.materialize(), 2 * nn),
    ]
    for name, fn, nbytes in cases:
        for _ in range(3):
            r = fn(); del r
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            r = fn(); del r
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        gbs = nbytes / (ms * 1e-3) / 1e9 if nbytes else 0.0
        print(json.dumps({"op": name, "n": n, "blk": blk, "ms": round(ms, 4), "algorithmic_bytes": nbytes,
                          "GBps": round(gbs, 1), "frac_of_measured_hbm": round(gbs / peak, 3), "hbm_peak_GBps": peak}))
    s.stop()
