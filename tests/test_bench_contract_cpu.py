"""bench.py restates the engine's residue-plane capacity rule to describe how many launches a step's GEMM takes: the two must
stay the same rule."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_plane_capacity_rule_is_the_engines():
    src = open(os.path.join(ROOT, "matrel_b200", "csrc", "abi_multiply.cpp")).read()
    assert re.search(r"plane_cap_tiles = std::max<int64_t>\(64, \(2ll << 30\) / \(static_cast<int64_t>\(T\) \* kOz2TileM \* kOz2TileN\)\)", src)
    assert "max_tiles += max_tiles & 1;" in src
    assert "constexpr int kOz2TileM = 128, kOz2TileN = 256;" in open(os.path.join(ROOT, "matrel_b200", "csrc", "kernels.h")).read()
    bench = open(os.path.join(ROOT, "bench.py")).read()
    assert "plane_cap = max(64, (2 << 30) // (max(1, moduli_used) * 128 * 256))" in bench
    assert "plane_cap += plane_cap & 1" in bench
