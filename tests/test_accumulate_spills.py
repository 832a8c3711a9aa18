"""k_accumulate of the BLS12-381 G1 ids keeps its whole mixed addition in registers: ptxas reports no stack frame and no
spill stores or loads, and the SASS holds no local-memory instruction.  The kernel is compiled on its own for sm_90a with
the product's flags (csrc/msm_body.cuh acc_blocks_per_sm: 3 blocks of 128 threads, <= 168 registers; the field products
inline).  A spill there costs local-memory traffic on every field multiplication of the MSM's hot loop."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "noble-curves_b200", "csrc")
NVCC = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DNMSM_MUL_NOINLINE", "-Xptxas", "-v"]
SRC = """#include "engine.cuh"
namespace nmsm {
template __global__ void k_accumulate<%s>(const uint32_t*, const uint32_t*, const uint32_t*, MsmPlan, uint32_t, uint32_t*,
                                          uint32_t*, uint32_t*);
}
"""


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
@pytest.mark.parametrize("curve", ["CurveBls381G1", "CurveBls381G1Any"])
def test_accumulate_has_no_local_memory(curve, tmp_path):
    src, obj = tmp_path / "acc.cu", tmp_path / "acc.o"
    src.write_text(SRC % curve)
    p = subprocess.run([NVCC] + FLAGS + ["-I", CSRC, "-c", str(src), "-o", str(obj)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-4000:]
    log = p.stdout + p.stderr
    # ptxas: "Compiling entry function '<mangled>'" ... "N bytes stack frame, N bytes spill stores, N bytes spill loads"
    entry = re.search(r"Compiling entry function '(_ZN4nmsm12k_accumulate[^']*)'.*?(\d+) bytes stack frame, (\d+) bytes "
                      r"spill stores, (\d+) bytes spill loads.*?Used (\d+) registers", log, re.S)
    assert entry, log[-4000:]
    name, stack, st, ld, regs = entry.group(1), *map(int, entry.groups()[1:])
    assert (stack, st, ld) == (0, 0, 0), "k_accumulate<%s>: %d B stack, %d B spill stores, %d B spill loads (%d registers)" % (
        curve, stack, st, ld, regs)
    assert regs <= 168  # 3 blocks of 128 threads per SM
    if os.path.exists(CUOBJDUMP):
        sass = subprocess.run([CUOBJDUMP, "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
        body = sass.split("Function : " + name, 1)[1].split("Function : ", 1)[0]
        assert not re.search(r"\b(LDL|STL)\b", body), "local-memory instructions in k_accumulate<%s>" % curve
