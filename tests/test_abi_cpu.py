"""CPU tests of the boundary: the C-ABI library loads, exports every symbol include/matrel.h
declares, the ctypes binding covers the same set, the integer placement functions are bit-exact
against the golden tables, and the engine refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import json
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(os.path.dirname(__file__), "golden")


def header_symbols():
    src = open(os.path.join(ROOT, "include", "matrel.h")).read()
    return sorted(set(re.findall(r"MR_API\s+[\w\s\*]+?\b(mr_\w+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    import matrel_b200._native as N
    syms = header_symbols()
    assert len(syms) >= 30
    out = subprocess.run(["nm", "-D", "--defined-only", N.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    for s in syms:
        assert s in exported, f"{s} declared in matrel.h but not exported by the .so"
        assert hasattr(N.lib, s)
    bound = set(N.SIGNATURES) | set(N._STR_FUNCS)
    assert bound == set(syms), (bound ^ set(syms))
    # nothing but the ABI (and nothing torch / C++-mangled) is exported
    extra = {e for e in exported if not e.startswith("mr_")}
    assert not extra, extra
    assert N.lib.mr_version().startswith(b"matrel-b200")


def test_library_is_not_older_than_its_sources():
    """The in-tree .so is what the package loads: a source or header edited after the last build would ship a stale ABI."""
    import glob
    import matrel_b200._native as N
    srcs = glob.glob(os.path.join(ROOT, "matrel_b200", "csrc", "*")) + [os.path.join(ROOT, "include", "matrel.h")]
    newest = max(srcs, key=os.path.getmtime)
    assert os.path.getmtime(N.LIB_PATH) >= os.path.getmtime(newest), f"{newest} is newer than the built library: run __graft_entry__.build()"


def test_stats_struct_matches_the_header():
    import matrel_b200._native as N
    src = open(os.path.join(ROOT, "include", "matrel.h")).read()
    body = re.search(r"typedef struct mr_stats \{(.*?)\} mr_stats;", src, re.S).group(1)
    fields = re.findall(r"^\s*(int64_t|double)\s+(\w+);", body, re.M)
    assert [(n, {"int64_t": C.c_int64, "double": C.c_double}[t]) for t, n in fields] == list(N.mr_stats._fields_)


def test_so_contains_hopper_native_sass():
    """UBLKCP / UTMALDG = TMA bulk and tensor copies, DMMA = fp64 tensor pipe, IGMMA / HGMMA = wgmma (s8 / tf32), SYNCS = mbarrier."""
    import matrel_b200._native as N
    sass = subprocess.run(["cuobjdump", "-sass", N.LIB_PATH], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", N.LIB_PATH], capture_output=True, text=True).stdout
    assert sass.count("DMMA") >= 128 and "UBLKCP" in sass and "UTMALDG" in sass and "SYNCS" in sass
    assert "IGMMA" in sass and "HGMMA" in sass


def test_partitioners_bit_exact():
    import matrel_b200 as mb
    g = json.load(open(os.path.join(G, "partitioners.json")))
    for c in g["cases"]:
        p = mb.genBlockCyclicPartitioner(c["nrows"], c["ncols"], c["blkSize"])
        assert list(p) == c["params"]
        bc = mb.BlockCyclicPartitioner(*p)
        assert bc.numPartitions == c["numPartitions"]
        used = set()
        for i in range(p[0]):
            for j in range(p[1]):
                v = bc.getPartition((i, j))
                used.add(v)
                if c["table"] is not None:
                    assert v == c["table"][i][j]
        assert sorted(used) == c["used"]
    for name, k in g["known"].items():
        n, blk = map(int, name.split("/"))
        assert list(mb.genBlockCyclicPartitioner(n, n, blk)) == k["params"]
    for i, p, want in g["row"]:
        assert mb.RowPartitioner(p).getPartition((i, 5)) == want
        assert mb.RowPartitioner(p).getPartition((i, 5, 9)) == want
    for j, p, want in g["col"]:
        assert mb.ColumnPartitioner(p).getPartition((5, j)) == want
    assert mb.IndexPartitioner(8).getPartition(5) == 5
    with pytest.raises(ValueError, match="Unrecognized key"):
        mb.RowPartitioner(4).getPartition("x")
    with pytest.raises(mb.IllegalArgumentException, match="Number of partitions cannot be negative but found -1"):
        mb.RowPartitioner(-1).getPartition((1, 1))
    with pytest.raises(mb.IllegalArgumentException, match="Number of row blocks should be larger than 0, but found 0"):
        mb.BlockCyclicPartitioner(0, 4, 1, 1)


def test_partitioners_match_oracle_exhaustively():
    import matrel_b200 as mb
    from oracle import matrel_oracle as O
    for R in range(1, 20):
        for Cc in (1, 2, 5, 16, 33):
            for r in (1, 2, 3, 8):
                for c in (1, 2, 4):
                    a, b = mb.BlockCyclicPartitioner(R, Cc, r, c), O.BlockCyclicPartitioner(R, Cc, r, c)
                    assert a.numPartitions == b.numPartitions
                    for i in range(R):
                        for j in range(Cc):
                            assert a.getPartition((i, j)) == b.getPartition(i, j)
    for nr in (1, 7, 100, 1000, 4096, 12345, 65536):
        for nc in (1, 9, 512, 3000, 65536):
            for blk in (1, 3, 100, 256, 1024):
                if nr // blk > 5000 or nc // blk > 5000:
                    continue
                assert tuple(mb.genBlockCyclicPartitioner(nr, nc, blk)) == O.gen_block_cyclic_partitioner(nr, nc, blk)


def test_partition_id_covers_the_four_schemes():
    """mr_partition_id (SURVEY 8b): the single placement entry point agrees with the per-scheme functions and the oracle."""
    from matrel_b200 import partitioner as P
    from oracle import matrel_oracle as O
    for i in range(0, 40, 3):
        for j in range(0, 40, 7):
            for p in (1, 2, 7, 8, 64):
                assert P.partition_id(P.PART_ROW, (p,), i, j) == O.row_partition(i, j, p)
                assert P.partition_id(P.PART_COLUMN, (p,), i, j) == O.column_partition(i, j, p)
                assert P.partition_id(P.PART_INDEX, (p,), i, j) == O.index_partition(i)
            params = O.gen_block_cyclic_partitioner(16384, 16384, 1024)
            assert P.partition_id(P.PART_BLOCK_CYCLIC, params, i, j) == O.BlockCyclicPartitioner(*params).getPartition(i, j)
    with pytest.raises(Exception, match="unknown partition scheme"):
        P.partition_id(9, (1,), 0, 0)


def test_no_cpu_fallback_without_gpu():
    """On a box without a CUDA device the engine must fail loudly, never compute on the host."""
    import torch
    import matrel_b200 as mb
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(mb.CudaError, match="no CPU fallback"):
        mb.MatfastSession()


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "matrel_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("the CPU oracle", ""), f


def test_cpp_facade_compiles():
    """include/matrel.hpp (C++ mirror of the Dataset API) compiles against the C ABI."""
    hpp = os.path.join(ROOT, "include", "matrel.hpp")
    if not os.path.exists(hpp):
        pytest.skip("no C++ facade yet")
    src = '#include "matrel.hpp"\nint main() { return 0; }\n'
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c++", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_jni_shim_type_checks_against_the_abi():
    """bindings/jni/matrel_jni.cpp cannot be built here (no JDK); with a stand-in <jni.h> that declares only what the shim uses
    (tests/cpp/jni_stub) g++ still checks every call it makes into include/matrel.h, so the shim cannot drift from the ABI."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Wextra", "-Wno-comment", "-Werror",
                        "-I", os.path.join(ROOT, "tests", "cpp", "jni_stub"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "bindings", "jni", "matrel_jni.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_header_is_plain_c():
    """include/matrel.h is consumable from C (the cgo / JNI / ctypes boundary): gcc -std=c99 parses it."""
    r = subprocess.run(["gcc", "-std=c99", "-fsyntax-only", "-Wall", "-Werror", "-x", "c", os.path.join(ROOT, "include", "matrel.h")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_scala_native_declarations_match_the_jni_shim():
    """Neither side of the JVM binding can be compiled here (no JDK, no scalac), so the two files are checked against each other:
    every `@native def` of bindings/scala/Dataset.scala has exactly one Java_..._Native_<name> in bindings/jni/matrel_jni.cpp with the
    same arity and the JNI type of every parameter and of the result, and the shim exports nothing the facade does not declare."""
    import re
    scala = open(os.path.join(ROOT, "bindings", "scala", "Dataset.scala")).read()
    jni = open(os.path.join(ROOT, "bindings", "jni", "matrel_jni.cpp")).read()
    to_jni = {"Long": "jlong", "Int": "jint", "Double": "jdouble", "Boolean": "jboolean", "Byte": "jbyte", "Unit": "void",
              "Array[Int]": "jintArray", "Array[Double]": "jdoubleArray", "Array[Long]": "jlongArray"}
    natives = {}
    for m in re.finditer(r"@native def (\w+)\(([^)]*)\)\s*:\s*([\w\[\]]+)", scala, re.S):
        params = [p.split(":")[1].strip() for p in m.group(2).split(",") if p.strip()]
        natives[m.group(1)] = ([to_jni[p] for p in params], to_jni[m.group(3)])
    # the shim generates some functions with macros: look at what the preprocessor makes of it (stand-in <jni.h> of tests/cpp/jni_stub)
    r = subprocess.run(["g++", "-std=c++17", "-E", "-P", "-I", os.path.join(ROOT, "tests", "cpp", "jni_stub"), "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "bindings", "jni", "matrel_jni.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    shim = {}
    for m in re.finditer(r"(\w+)\s+Java_org_apache_spark_sql_matfast_b200_Native_(\w+)\s*\(\s*JNIEnv\s*\*\s*\w*\s*,\s*jclass\s*((?:,[^)]*)?)\)\s*\{",
                         r.stdout, re.S):
        args = [a.strip().rsplit(" ", 1)[0].strip() for a in m.group(3).split(",") if a.strip()]
        assert m.group(2) not in shim, f"{m.group(2)} defined twice in the shim"
        shim[m.group(2)] = (args, m.group(1))
    assert len(natives) >= 45 and set(natives) == set(shim), (sorted(set(natives) - set(shim)), sorted(set(shim) - set(natives)))
    for name, sig in natives.items():
        assert sig == shim[name], (name, sig, shim[name])
    # the package path of the exported symbols is the one the facade's `object Native` lives in
    assert "Java_org_apache_spark_sql_matfast_b200_Native_##NAME" in jni and "package org.apache.spark.sql.matfast.b200" in scala


REFERENCE_DATASET_METHODS = ["project", "selection", "t", "transpose", "rowSum", "colSum", "sum", "trace", "vec", "addScalar",
                             "multiplyScalar", "power", "addElement", "multiplyElement", "divideElement", "matrixMultiply",
                             "matrixRankOneUpdate"]   # M/Dataset.scala:38-152, in source order


def test_facades_expose_the_reference_operator_names():
    """The three host-side mirrors of the reference's Dataset (Python, C++, Scala) carry every public operator name of
    M/Dataset.scala:38-152; the grid classes carry all but vec / matrixRankOneUpdate (DESIGN.md section 5)."""
    import re
    import matrel_b200 as mb
    for name in REFERENCE_DATASET_METHODS:
        assert callable(getattr(mb.Dataset, name)), name
    hpp = open(os.path.join(ROOT, "include", "matrel.hpp")).read()
    scala = open(os.path.join(ROOT, "bindings", "scala", "Dataset.scala")).read()
    cls_hpp = hpp[hpp.index("class Dataset {"):hpp.index("class GridSession")]
    grid_hpp = hpp[hpp.index("class DistributedDataset {"):]
    cls_scala = scala[scala.index("class B200Dataset"):scala.index("class B200GridSession")]
    grid_scala = scala[scala.index("class B200GridDataset"):]
    for name in REFERENCE_DATASET_METHODS:
        assert re.search(r"\b%s\(" % name, cls_hpp), f"matrel.hpp Dataset lacks {name}"
        assert re.search(r"def %s\(" % name, cls_scala), f"B200Dataset lacks {name}"
        if name not in ("vec", "matrixRankOneUpdate"):
            assert re.search(r"\b%s\(" % name, grid_hpp), f"matrel.hpp DistributedDataset lacks {name}"
            assert re.search(r"def %s\(" % name, grid_scala), f"B200GridDataset lacks {name}"
    for extra in ("collect", "getBlock"):
        assert re.search(r"def %s\(" % extra, cls_scala) and re.search(r"def %s\(" % extra, grid_scala), extra
