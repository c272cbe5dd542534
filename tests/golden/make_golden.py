"""Generates tests/golden/*.json.

The reference has no tests and cannot run here (no JVM), so there are no reference-produced
vectors to import.  What the reference DOES fix are the inputs of its println demos and the
matrix pictures in their comments.  This script writes those inputs down verbatim and derives the
expected outputs with plain dense numpy arithmetic on the full (un-blocked) matrices -- it does
NOT import the oracle or the product, so it is an independent pin for both.

Sources (paths under <reference>/src/main/scala/org/apache/spark/sql/matfast/):
  example/BasicMatrixOps.scala:107-144   b1..b4, s1, mat1, mat2 and their pictures
  matrix/LocalMatrix.scala:1096-1135     TestSparse: spmat1, spmat2, den1, den2, denV
  partitioner/*.scala, execution/MatfastExecutionHelper.scala:46-62   partitioner formulas

Run:  python tests/golden/make_golden.py
"""
import json
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def colmajor(a):
    return [float(x) for x in np.asarray(a, dtype=float).T.reshape(-1)]


def basic_matrix_ops():
    # BasicMatrixOps.scala:109-116 (values are column-major 2x2)
    blocks = {
        "b1": {"type": "dense", "numRows": 2, "numCols": 2, "values": [1, 1, 2, 2]},
        "b2": {"type": "dense", "numRows": 2, "numCols": 2, "values": [2, 2, 3, 3]},
        "b3": {"type": "dense", "numRows": 2, "numCols": 2, "values": [3, 3, 4, 4]},
        "b4": {"type": "dense", "numRows": 2, "numCols": 2, "values": [4, 5, 6, 7]},
        "s1": {"type": "sparse", "numRows": 2, "numCols": 2, "colPtrs": [0, 1, 2], "rowIndices": [1, 0],
               "values": [4, 2]},
    }
    mat1 = [[0, 0, "b1"], [1, 1, "b2"]]
    mat2 = [[0, 0, "b3"], [0, 1, "b4"], [1, 1, "s1"]]
    # the pictures at BasicMatrixOps.scala:127-144, typed in as full matrices
    M1 = np.array([[1, 2, 0, 0], [1, 2, 0, 0], [0, 0, 2, 3], [0, 0, 2, 3]], dtype=float)
    M2 = np.array([[3, 4, 4, 6], [3, 4, 5, 7], [0, 0, 0, 2], [0, 0, 4, 0]], dtype=float)
    P = M1 @ M2
    present1 = {(0, 0), (1, 1)}
    present2 = {(0, 0), (0, 1), (1, 1)}
    prod_blocks = {}
    for i in range(2):
        for j in range(2):
            if any((i, k) in present1 and (k, j) in present2 for k in range(2)):
                prod_blocks[f"{i},{j}"] = colmajor(P[2 * i:2 * i + 2, 2 * j:2 * j + 2])
    S = M1 + M2
    return {
        "source": "example/BasicMatrixOps.scala:107-144",
        "blkSize": 2, "nrows": 4, "ncols": 4,
        "blocks": blocks, "mat1": mat1, "mat2": mat2,
        "expected": {
            # matrixMultiply(4, 4, mat2, 4, 4, 2) (:118); block (1,0) has no matching k -> absent
            "multiply_blocks_colmajor": prod_blocks,
            "multiply_absent": ["1,0"],
            "multiply_full": P.tolist(),
            "trace": float(np.trace(P)),                      # :174
            "selection_0_3": float(P[0, 3]),                  # :234
            "column_3": [float(x) for x in P[:, 3]],          # :212
            "rowSum_mat1_t": [float(x) for x in M1.T.sum(axis=1)],   # :159
            "colSum_mat2": [float(x) for x in M2.sum(axis=0)],       # :166
            # addElement: outer join, every key of either side present
            "add_full": S.tolist(),
            "add_present": ["0,0", "0,1", "1,1"],
            # multiplyElement: inner join, keys on both sides only
            "mul_full_on_common": (M1 * M2).tolist(),
            "mul_present": ["0,0", "1,1"],
            "transpose_mat1_full": M1.T.tolist(),
            # runMatrixProjection (:196, :204): row 2 of mat1 as 1 x 4, column 3 of mat2 as 4 x 1
            "project_row_2_mat1": [float(x) for x in M1[2, :]],
            "project_col_3_mat2": [float(x) for x in M2[:, 3]],
        },
        # runMatrixTranspose (:47-64): blocks at ids (0,2) s1, (2,3) b2, (4,5) b3, (6,7) b4; t() swaps the ids and flips flags
        "transpose_demo": {
            "blocks": [[0, 2, "s1"], [2, 3, "b2"], [4, 5, "b3"], [6, 7, "b4"]],
            "expected": {"2,0": np.array([[0, 2], [4, 0]], dtype=float).T.tolist(),     # s1 = [[0,2],[4,0]]
                         "3,2": np.array([[2, 3], [2, 3]], dtype=float).T.tolist(),
                         "5,4": np.array([[3, 4], [3, 4]], dtype=float).T.tolist(),
                         "7,6": np.array([[4, 6], [5, 7]], dtype=float).T.tolist()},
        },
        # runMatrixScalar (:66-78): power(2) of b1 at (0,2) and s1 at (1,3); element-wise squares, structure kept
        "power_demo": {
            "blocks": [[0, 2, "b1"], [1, 3, "s1"]],
            "expected": {"0,2": (np.array([[1, 2], [1, 2]], dtype=float) ** 2).tolist(),
                         "1,3": (np.array([[0, 2], [4, 0]], dtype=float) ** 2).tolist()},
        },
    }


def test_sparse():
    # LocalMatrix.scala:1098-1105
    sp1 = {"numRows": 3, "numCols": 3, "colPtrs": [0, 2, 3, 6], "rowIndices": [0, 2, 1, 0, 1, 2],
           "values": [1, 2, 3, 4, 5, 6]}
    sp2 = {"numRows": 3, "numCols": 3, "colPtrs": [0, 1, 3, 4], "rowIndices": [1, 0, 2, 0], "values": [3, 1, 2, 2]}
    S1 = np.array([[1, 0, 4], [0, 3, 5], [2, 0, 6]], dtype=float)   # the CSC arrays above, written out
    S2 = np.array([[0, 1, 2], [3, 0, 0], [0, 2, 0]], dtype=float)
    v = np.array([1, 2, 3], dtype=float)
    return {
        "source": "matrix/LocalMatrix.scala:1096-1135 (TestSparse)",
        "spmat1": sp1, "spmat2": sp2,
        "S1_full": S1.tolist(), "S2_full": S2.tolist(),
        "denV": [1, 2, 3],
        "den1_colmajor": [1, 4, 7, 2, 5, 8, 3, 6, 9], "den2_colmajor": [1, 2, 3, 1, 2, 3, 1, 2, 3],
        "expected": {
            "S1_times_S2": (S1 @ S2).tolist(),             # multiplySparseSparse(spmat1, spmat2) :1112
            "S1_hadamard_S2": (S1 * S2).tolist(),          # elementWiseMultiply :1114
            "S1_plus_S2": (S1 + S2).tolist(),              # add :1116
            "S2_times_S2t": (S2 @ S2.T).tolist(),          # incrementalMultiply(spmat2, spmat2.transpose, 0) :1126
            "S1_times_v": (S1 @ v).tolist(),               # multiplySparseMatDenseVec :1130
            "S1_times_S2t": (S1 @ S2.T).tolist(),          # :1132
        },
    }


def partitioners():
    def jround(x):
        return int(math.floor(x + 0.5))

    def gen(nrows, ncols, blk):   # MatfastExecutionHelper.scala:46-62, transcribed
        R = int(math.ceil(nrows * 1.0 / blk))
        Cc = int(math.ceil(ncols * 1.0 / blk))
        r = jround(max(R / 8.0, 1.0))
        c = jround(max(Cc / 8.0, 1.0))
        if r == 1 or c == 1:
            if r != 1:
                r = jround(max(r / 8.0, 1.0))
            if c != 1:
                c = jround(max(c / 8.0, 1.0))
        return [R, Cc, r, c]

    def table(p):                 # BlockCyclicPartitioner.scala:46-58, transcribed
        R, Cc, r, c = p
        rpn = int(math.ceil(R * 1.0 / r))
        cpn = int(math.ceil(Cc * 1.0 / c))
        nrp, ncp = R // rpn, Cc // cpn
        n = rpn * cpn
        return n, [[((i % nrp) * cpn + (j % ncp)) % n for j in range(Cc)] for i in range(R)]

    cases = []
    for (nr, nc, blk) in [(1024, 1024, 256), (4096, 4096, 512), (16384, 16384, 1024), (65536, 65536, 2048),
                          (32768, 32768, 1024), (4, 4, 2), (1000, 3000, 100), (100, 12800, 100), (10, 10, 3),
                          (20000, 100, 100)]:
        p = gen(nr, nc, blk)
        n, tab = table(p)
        cases.append({"nrows": nr, "ncols": nc, "blkSize": blk, "params": p, "numPartitions": n,
                      "used": sorted({x for row in tab for x in row}), "table": tab if p[0] * p[1] <= 1024 else None})
    return {
        "source": "partitioner/BlockCyclicPartitioner.scala:46-58, execution/MatfastExecutionHelper.scala:46-62",
        # SURVEY.md section 8(a13) known answers
        "known": {"1024/256": {"params": [4, 4, 1, 1], "n": 16, "used": [0]},
                  "4096/512": {"params": [8, 8, 1, 1], "n": 64, "used": [0]},
                  "16384/1024": {"params": [16, 16, 2, 2], "n": 64, "used": [0, 1, 8, 9]},
                  "65536/2048": {"params": [32, 32, 4, 4], "n": 64,
                                 "used": [0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 19, 24, 25, 26, 27]}},
        "cases": cases,
        "row": [[i, p, i % p] for i in range(0, 40, 3) for p in (1, 2, 7, 8, 64)],
        "col": [[j, p, j % p] for j in range(0, 40, 3) for p in (1, 2, 7, 8, 64)],
    }


def java_random():
    # java.util.Random known answers (JDK documentation / widely published): seed 42 first nextInt() is
    # -1170105035 and first nextDouble() of a fresh Random(42) is 0.7275636800328681; seed 0 first
    # nextInt() is -1155484576, first nextDouble() of Random(0) is 0.730967787376657.
    return {"source": "java.util.Random (JDK), known answers",
            "nextInt": {"42": -1170105035, "0": -1155484576},
            "nextDouble": {"42": 0.7275636800328681, "0": 0.730967787376657}}


if __name__ == "__main__":
    for name, obj in [("basic_matrix_ops", basic_matrix_ops()), ("test_sparse", test_sparse()),
                      ("partitioners", partitioners()), ("java_random", java_random())]:
        with open(os.path.join(HERE, name + ".json"), "w") as f:
            json.dump(obj, f, indent=1)
        print("wrote", name)
