"""Timing of matrix x vector products (DESIGN section 4.5.5): whole matrixMultiply calls timed with CUDA events and a synchronise,
the median of 5 after a warm-up, at blk 1024.  One JSON line per case.

  dense:  A x and x^T A at N in --dense-sizes, column-major (rand) and row-major (t() of rand) blocks, alternating in the same
          session with the same product under gemm_algo 1 (for dense pairs exactly the DMMA route that ran before the vector route).
  sparse: sprand at N in --sparse-sizes, densities 1e-4 / 1e-3 / 1e-2, CSR and CSC: S x, t(S) x, x^T S, and a 20-step iteration
          x <- S x scaled with multiplyScalar each step.  --root DIR imports the package from another tree (a build of an earlier
          commit) to time its routes on the same operands; "does not fit" where that route's dense images exceed the card.
  --save FILE / --compare FILE: store the outputs, or compare them with stored ones (max |difference| / max |value|).
  --cols T (default 1): a thin side of T columns (A X) or rows (X^T A) instead of one vector: X is fromDense of a C-order N x T
          array and X^T its t().  Each product alternates in the same session with the T width-1 products of its columns
          ("width1_ms"; "same_bits_as_width1" compares the bits) and, for dense A, with itself under gemm_algo 1.

Rates are compulsory bytes (the stored matrix, X and C, once) over time, against the 3.35 TB/s HBM3 data-sheet figure of the
H100 SXM; that figure is a data-sheet number, not a measured one."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--dense-sizes", default="16384,32768,65536")
ap.add_argument("--sparse-sizes", default="32768,131072")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--save")
ap.add_argument("--compare")
ap.add_argument("--cols", type=int, default=1)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

import matrel_b200 as mb  # noqa: E402
from matrel_b200 import _native  # noqa: E402
from matrel_b200.dataset import sprand  # noqa: E402

BLK = 1024
DATASHEET_BPS = 3.35e12
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
saved = {}
stored = dict(np.load(args.compare)) if args.compare else None


def timed(s, fn):
    fn()
    s.sync()
    ms = []
    out = None
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        s.sync()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), out


def vector(s, x, row):
    n = x.size
    return s.createDataset(mb.MatrixBlock(0 if row else b, b if row else 0,
                                          mb.DenseMatrix.from_numpy(x[b * BLK:(b + 1) * BLK][None, :] if row else x[b * BLK:(b + 1) * BLK, None]))
                           for b in range(-(-n // BLK)))


T = args.cols


def thin(s, x):
    """(X, X^T) for an N x T array: fromDense of its C-order copy (row-major blocks) and the t() of that."""
    X = s.fromDense(np.ascontiguousarray(x), BLK)
    return X, X.t()


def width1(s, x, call):
    """The T width-1 products of the columns of x, one call each: call(vector dataset) -> result dataset."""
    cols = [(vector(s, x[:, j], False), vector(s, x[:, j], True)) for j in range(T)]
    return lambda row: [call(c[1] if row else c[0]) for c in cols]


def same_as_width1(C, outs, n, row):
    a = C.toNumpy(T if row else n, n if row else T, BLK)
    return all(np.array_equal((a[j] if row else a[:, j]).view(np.int64),
                              o.toNumpy(1 if row else n, n if row else 1, BLK).reshape(-1).view(np.int64)) for j, o in enumerate(outs))


def emit(rec, name, ds, n, row):
    v = ds.toNumpy(T if row else n, n if row else T, BLK).reshape(-1)
    key = f"{name}" if T == 1 else f"{name}-cols{T}"
    saved[key] = v
    if stored is not None and key in stored:
        w = stored[key]
        scale = float(np.abs(w).max()) or 1.0
        rec["max_rel_diff_vs_stored"] = float(np.abs(v - w).max() / scale)
    if T > 1:
        rec["cols"] = T
    rec["card"] = card
    print(json.dumps(rec), flush=True)


def stats(s):
    st = s.stats()
    return {"mv_pairs": st["mv_pairs"] // (args.reps + 1), "kernel_launches": st["kernel_launches"] // (args.reps + 1)}  # per call


with mb.MatfastSession(device=0) as s:
    has_mv = "mv_pairs" in dict(_native.mr_stats._fields_)   # False for a build from before the vector route

    def probe():   # does X^T S with T rows take the stored-entry route (no dense images) in this build?
        if not has_mv:
            return False
        P = sprand(s, 64, 64, 64, 0.1, 1, csr=True)
        s.reset_stats()
        (vector(s, np.ones(64), True) if T == 1 else thin(s, np.ones((64, T)))[1]).matrixMultiply(T, 64, P, 64, 64, 64)
        s.sync()
        return s.stats()["mv_pairs"] > 0
    thin_route = probe()
    for N in [int(t) for t in args.dense_sizes.split(",") if t]:
        A = s.rand(N, N, BLK, 1)
        for layout, M in (("col", A), ("row", A.t())):
            x = np.random.default_rng(N).uniform(-1, 1, N if T == 1 else (N, T))
            for form in ("Ax", "xA"):
                row = form == "xA"
                X = vector(s, x, row) if T == 1 else thin(s, x)[row]
                call = (lambda: M.matrixMultiply(N, N, X, N, T, BLK)) if form == "Ax" else (lambda: X.matrixMultiply(T, N, M, N, N, BLK))
                one = None if T == 1 else width1(s, x, (lambda v: v.matrixMultiply(1, N, M, N, N, BLK)) if row else
                                                 (lambda v: M.matrixMultiply(N, N, v, N, 1, BLK)))
                for algo in (0, 1, 0, 1):   # alternating; the second of each pair is reported
                    s.set_option("gemm_algo", algo)
                    s.reset_stats()
                    ms, C = timed(s, call)
                    st = s.stats()
                    if algo == 0:
                        ms0, C0, st0 = ms, C, st
                        if one is not None:
                            msw, outs = timed(s, lambda: one(row))
                    else:
                        ms1, C1 = ms, C
                s.set_option("gemm_algo", 0)
                nbytes = 8.0 * (N * N + 2 * N * T)
                rec = {"case": "dense", "N": N, "layout": layout, "form": form, "ms": ms0, "gemm_algo1_ms": ms1,
                       "bytes_per_s": nbytes / (ms0 * 1e-3), "share_of_datasheet_bw": nbytes / (ms0 * 1e-3) / DATASHEET_BPS,
                       "mv_pairs": st0["mv_pairs"] if has_mv else None}
                if one is not None:
                    rec.update({"width1_ms": msw, "same_bits_as_width1": same_as_width1(C0, outs, N, row)})
                    del outs
                a0 = C0.toNumpy(T if row else N, N if row else T, BLK).reshape(-1)
                a1 = C1.toNumpy(T if row else N, N if row else T, BLK).reshape(-1)
                rec["max_rel_diff_vs_gemm_algo1"] = float(np.abs(a0 - a1).max() / np.abs(a1).max())
                emit(rec, f"dense-{N}-{layout}-{form}", C0, N, form == "xA")
                del X, C0, C1
        del A, M
    free = torch.cuda.mem_get_info()[1]
    for N in [int(t) for t in args.sparse_sizes.split(",") if t]:
        nb = N // BLK
        for d in (1e-4, 1e-3, 1e-2):
            for csr in (True, False):
                S = sprand(s, N, N, BLK, d, 7, csr=csr)
                nnz = d * N * N   # sprand stores round(density * blk^2) distinct entries per block
                x = np.random.default_rng(N + 1).uniform(-1, 1, N if T == 1 else (N, T))
                Xc, Xr = (vector(s, x, False), vector(s, x, True)) if T == 1 else thin(s, x)
                St = S.t()
                for form, call, row, images in (("Sx", lambda: S.matrixMultiply(N, N, Xc, N, T, BLK), False, 0),
                                                ("tSx", lambda: St.matrixMultiply(N, N, Xc, N, T, BLK), False, 0),
                                                ("xS", lambda: Xr.matrixMultiply(T, N, S, N, N, BLK), True, nb * nb * BLK * BLK * 8)):
                    rec = {"case": "sprand", "N": N, "density": d, "format": "csr" if csr else "csc", "form": form}
                    if not thin_route and images > free:
                        rec.update({"ms": None, "note": f"does not fit: {images / 2**30:.0f} GiB of dense images"})
                        rec["card"] = card
                        print(json.dumps(rec), flush=True)
                        continue
                    s.reset_stats()
                    ms, C = timed(s, call)
                    nbytes = 12.0 * nnz + 4.0 * (N + nb) * nb + 8.0 * N * (T + 1)
                    rec.update({"ms": ms, "bytes_per_s": nbytes / (ms * 1e-3), "share_of_datasheet_bw": nbytes / (ms * 1e-3) / DATASHEET_BPS,
                                **(stats(s) if has_mv else {})})
                    if T > 1:
                        M = St if form == "tSx" else S
                        one = width1(s, x, (lambda v: v.matrixMultiply(1, N, M, N, N, BLK)) if row else
                                     (lambda v: M.matrixMultiply(N, N, v, N, 1, BLK)))
                        msw, outs = timed(s, lambda: one(row))
                        rec.update({"width1_ms": msw, "same_bits_as_width1": same_as_width1(C, outs, N, row)})
                        del outs
                    emit(rec, f"sprand-{N}-{d:g}-{rec['format']}-{form}", C, N, row)
                    del C

                def iterate():
                    v = Xc
                    for _ in range(20):
                        v = S.matrixMultiply(N, N, v, N, T, BLK).multiplyScalar(0.5)
                    return v
                ms, V = timed(s, iterate)
                rec = {"case": "sprand-iterate-20", "N": N, "density": d, "format": "csr" if csr else "csc", "ms": ms}
                emit(rec, f"iter-{N}-{d:g}-{rec['format']}", V, N, False)
                del S, St, Xc, Xr, V
if args.save:
    np.savez(args.save, **saved)
