"""Spill bytes of the fp16 row owners of k_head_v2, inference and training instantiations, from the compiler's own report.

The fp16 owners run at 152 registers and still spill a little of their per-batch state (DESIGN §5). Writing the unsplit M-half
epilogues with stmatrix took those spills from 132 / 136 B to 92 / 92 B (inference) and from 160 / 160 B to 116 / 116 B
(training); these bounds keep them from creeping back. Compiling head_v2_kernel.cu for sm_90a with `-Xptxas=-v` needs nvcc,
not a GPU.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "genefaceplusplus_b200", "csrc", "head_v2_kernel.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

# (spill stores, spill loads) in bytes, at most
LIMITS = {
    "_ZN4gfpp9k_head_v2ILb0ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (92, 92),      # fp16 inference (the benchmarked kernel)
    "_ZN4gfpp15k_head_v2_trainILb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (116, 116),  # fp16 frozen head of the torso steps
    "_ZN4gfpp15k_head_v2_trainILb1EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (0, 0),      # robust frozen head
}


@pytest.fixture(scope="module")
def ptxas_report():
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                            "-Xptxas=-v", "-c", SRC, "-o", os.path.join(d, "v2.o")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    return r.stderr


@pytest.mark.parametrize("mangled", sorted(LIMITS))
def test_owner_spills_at_most(ptxas_report, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  ptxas_report)
    assert m, f"no ptxas report for {mangled}"
    st, ld = int(m.group(1)), int(m.group(2))
    lim_st, lim_ld = LIMITS[mangled]
    assert st <= lim_st and ld <= lim_ld, f"{mangled}: {st} / {ld} bytes of spill stores / loads (limit {lim_st} / {lim_ld})"
