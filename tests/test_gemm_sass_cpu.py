"""Guards on the machine code of the Ozaki-II CTA-pair GEMM (ozaki2_gemm_2sm_kernel, both work-item orders), read from the
built library with cuobjdump.

- The consumer warps hand every ring stage back to both CTAs of the pair with remote mbarrier arrivals.  Between the first
  wgmma (IGMMA) and the last of those arrivals there must be no GPU-scope memory barrier: a release.cluster arrive makes
  ptxas put MEMBAR.ALL.GPU in front of each one, on the critical path of every K stage.
- The residue epilogue reduces the s32 accumulators with integer arithmetic only: no fp64 multiply and no int <-> fp64
  conversion (those issue at a quarter of the ALU rate) anywhere in the kernel.

Skipped when cuobjdump or the built library is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "matrel_b200", "libmatrel_b200.so")
KERNEL = "ozaki2_gemm_2sm_kernel"


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def kernel_sass(lib, name):
    """{mangled function name: [instruction text, ...]} for every function of `lib` whose name contains `name`."""
    out = subprocess.run([_cuobjdump(), "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for part in re.split(r"\n\s*Function : ", out)[1:]:
        fname, body = part.split("\n", 1)
        if name not in fname:
            continue
        funcs[fname.strip()] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*;)", body)]
    return funcs


def fences_between_wgmma_and_release(ins):
    first = next(i for i, s in enumerate(ins) if "IGMMA" in s)
    last = max(i for i, s in enumerate(ins) if s.startswith("SYNCS.ARRIVE") and ".RED" in s)
    assert first < last
    return [s for s in ins[first:last + 1] if re.match(r"MEMBAR\.\S*GPU", s)]


def fp64_conversions(ins):
    return [s for s in ins if re.match(r"(I2F\.F64|F2I\S*\.F64|DMUL)\b", s)]


@pytest.fixture(scope="module")
def pair_kernels():
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    funcs = kernel_sass(LIB, KERNEL)
    insts = {f: ins for f, ins in funcs.items() if re.search(KERNEL + r"ILb[01]E", f)}
    assert len(insts) == 2, sorted(funcs)  # KSPLIT = false and true
    return insts


def test_stage_release_has_no_gpu_fence(pair_kernels):
    for f, ins in pair_kernels.items():
        assert fences_between_wgmma_and_release(ins) == [], f


def test_residue_epilogue_has_no_fp64_conversions(pair_kernels):
    for f, ins in pair_kernels.items():
        assert fp64_conversions(ins) == [], f
