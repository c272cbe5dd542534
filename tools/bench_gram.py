"""Timing of Gram products (DESIGN section 4.1.2): C = A A^T and C = A^T A through the Gram route (A and A.t() share their arrays),
alternating in the same session with the general route on a copy of A (A.multiplyScalar(1.0): the same bits in other arrays).
Whole matrixMultiply calls are timed with CUDA events and a synchronise; median of --reps after a warm-up of each.  Every timed
shape asserts that both routes give identical bits.  One JSON line per case, with the card, its power limit and max SM clock.

  AAt:      A A^T, A 16384 x 16384, blk 1024 (the bench.py shape), auto engine (Ozaki-II)
  AtA:      A^T A, A 32768 x 16384, blk 1024, auto
  XtX:      X^T X, X 262144 x 2048, blk 1024: K >= 2^17, so DMMA computes 3 of the 4 blocks
  AAt_dmma: A A^T as AAt under gemm_algo 1

Sparse cases (every block low-density sparse: the sparse x sparse chains, DESIGN section 4.5.1), blk 1024, A N x N from sprand
with CSR or CSC blocks; the general route runs on a copy of A re-ingested from its collected blocks:
  sp_{AAt,AtA}_{1e-3,1.3e-2}_{csr,csc}: N = 32768 at density 1e-3 (the chains end sparse) and 1.3e-2 (they end dense)
  sp_AAt_65536:  A A^T, N = 65536 at 1e-3, CSR
  sp_one_8192:   A A^T of one 8192 x 8192 CSR block at 1e-3, built on the host from a seeded generator (device sprand is limited
                 to about 14000 entries per block); only the diagonal triangle is saved here

The mirror kernel's time comes from a separate torch.profiler run of one Gram call; its rate is the bytes it moves (every
strictly-lower element read once and written once) over that time, against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM
(a data-sheet number, not a measured one)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--cases", default="AAt,AtA,XtX,AAt_dmma")  # or "sparse" for every sparse case
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import matrel_b200 as mb  # noqa: E402

BLK = 1024
DATASHEET_BPS = 3.35e12
CASES = {"AAt": ("AAt", 16384, 16384, 0), "AtA": ("AtA", 32768, 16384, 0), "XtX": ("AtA", 262144, 2048, 0),
         "AAt_dmma": ("AAt", 16384, 16384, 1)}
SPARSE = {f"sp_{kind}_{d}_{fmt}": (kind, 32768, float(d), fmt == "csr") for kind in ("AAt", "AtA") for d in ("1e-3", "1.3e-2")
          for fmt in ("csr", "csc")}
SPARSE["sp_AAt_65536"] = ("AAt", 65536, 1e-3, True)
SPARSE["sp_one_8192"] = ("AAt", 8192, 1e-3, True)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()


def timed_call(s, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.sync()
    e0.record()
    out = fn()
    s.sync()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def mirror_ms(s, fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        s.sync()
        torch.cuda.synchronize()
    del out
    us = sum(e.device_time_total for e in prof.events() if "gram_mirror" in e.name)
    return us / 1e3 if us > 0 else None


def run_case(s, name):
    kind, m, n, algo = CASES[name]
    s.set_option("gemm_algo", algo)
    A = s.rand(m, n, BLK, 42)
    A2 = A.multiplyScalar(1.0)
    if kind == "AAt":
        N, gram, general = m, (lambda: A.matrixMultiply(m, n, A.t(), n, m, BLK)), (lambda: A.matrixMultiply(m, n, A2.t(), n, m, BLK))
    else:
        N, gram, general = n, (lambda: A.t().matrixMultiply(n, m, A, m, n, BLK)), (lambda: A2.t().matrixMultiply(n, m, A, m, n, BLK))
    for fn in (gram, general):   # warm-up
        fn()
    s.sync()
    s.reset_stats()
    Cg = gram()
    s.sync()
    st = s.stats()
    assert st["gram_blocks"] > 0, st
    Cr = general()
    s.sync()
    assert s.stats()["gram_blocks"] == 0
    same = np.array_equal(Cg.toNumpy(N, N, BLK).view(np.int64), Cr.toNumpy(N, N, BLK).view(np.int64))
    assert same, f"{name}: the Gram route differs from the general route"
    del Cg, Cr
    tg, tr = [], []
    for _ in range(args.reps):
        t, C = timed_call(s, gram)
        tg.append(t)
        del C
        t, C = timed_call(s, general)
        tr.append(t)
        del C
    mir = mirror_ms(s, gram)
    nb = -(-N // BLK)
    lower = N * (N - 1) // 2
    rec = {"case": name, "C": f"{N}x{N}", "K": m if kind == "AtA" else n, "blk": BLK, "gemm_algo": algo,
           "gram_ms": float(np.median(tg)), "general_ms": float(np.median(tr)), "speedup": float(np.median(tr) / np.median(tg)),
           "gram_blocks": st["gram_blocks"], "gram_mirrored_blocks": st["gram_mirrored_blocks"], "output_blocks": nb * nb,
           "tc_int8_ops": st["tc_int8_ops"], "same_bits": bool(same), "mirror_ms": mir,
           "mirror_TBps": (16 * lower / (mir * 1e-3) / 1e12) if mir else None,
           "mirror_of_datasheet_bw": (16 * lower / (mir * 1e-3) / DATASHEET_BPS) if mir else None,
           "gram_ms_all": tg, "general_ms_all": tr, "card": card}
    s.set_option("gemm_algo", 0)
    return rec


def blocks_of(C):
    out = {}
    for b in C.collect():
        m = b.matrix
        sp = isinstance(m, mb.SparseMatrix)
        out[(b.rid, b.cid)] = (sp, m.isTransposed, m.numRows, m.numCols, m.values.view(np.int64).copy(),
                               m.colPtrs.copy() if sp else None, m.rowIndices.copy() if sp else None)
    return out


def same_blocks(x, y):
    if sorted(x) != sorted(y):
        return False
    for k, a in x.items():
        b = y[k]
        if a[:4] != b[:4]:
            return False
        for u, v in zip(a[4:], b[4:]):
            if (u is None) != (v is None) or (u is not None and not np.array_equal(u, v)):
                return False
    return True


def run_sparse_case(s, name):
    kind, N, density, csr = SPARSE[name]
    blk = BLK
    if name == "sp_one_8192":
        import scipy.sparse as sps
        blk = N
        a = sps.random(N, N, density=density, format="csr", random_state=np.random.default_rng(7), dtype=np.float64)
        a.sort_indices()
        A = s.createDataset([mb.MatrixBlock(0, 0, mb.SparseMatrix(N, N, a.indptr, a.indices, a.data, True))])
    else:
        A = mb.dataset.sprand(s, N, N, blk, density, 42, csr=csr)
    A2 = s.createDataset(A.collect())   # the same blocks in other arrays
    if kind == "AAt":
        gram, general = (lambda: A.matrixMultiply(N, N, A.t(), N, N, blk)), (lambda: A.matrixMultiply(N, N, A2.t(), N, N, blk))
    else:
        gram, general = (lambda: A.t().matrixMultiply(N, N, A, N, N, blk)), (lambda: A2.t().matrixMultiply(N, N, A, N, N, blk))
    for fn in (gram, general):   # warm-up
        fn()
    s.sync()
    s.reset_stats()
    Cg = gram()
    s.sync()
    st = s.stats()
    assert st["gram_blocks"] > 0, st
    Cr = general()
    s.sync()
    st_r = s.stats()
    assert st_r["gram_blocks"] == 0
    bg, br = blocks_of(Cg), blocks_of(Cr)
    same = same_blocks(bg, br)
    assert same, f"{name}: the Gram route differs from the general route"
    kinds = {"dense": sum(not v[0] for v in bg.values()), "sparse": sum(v[0] for v in bg.values())}
    del Cg, Cr, bg, br
    tg, tr = [], []
    for _ in range(args.reps):
        t, C = timed_call(s, gram)
        tg.append(t)
        del C
        t, C = timed_call(s, general)
        tr.append(t)
        del C
    return {"case": name, "C": f"{N}x{N}", "density": density, "blocks": "csr" if csr else "csc", "blk": blk,
            "gram_ms": float(np.median(tg)), "general_ms": float(np.median(tr)), "speedup": float(np.median(tr) / np.median(tg)),
            "gram_blocks": st["gram_blocks"], "gram_mirrored_blocks": st["gram_mirrored_blocks"], "output_kinds": kinds,
            "spgemm_products": st["spgemm_products"], "general_spgemm_products": st_r["spgemm_products"],
            "same_bits": bool(same), "gram_ms_all": tg, "general_ms_all": tr, "card": card}


with mb.MatfastSession(device=0) as s:
    names = [n for c in args.cases.split(",") for n in (SPARSE if c == "sparse" else [c])]
    for name in names:
        rec = run_sparse_case(s, name) if name in SPARSE else run_case(s, name)
        line = json.dumps(rec)
        print(line, flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")
