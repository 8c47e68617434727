"""Register budget of the row-owner head kernel (k_head_v2), checked from the compiler's own report.

The owner program's live set sits close to its register budget (setmaxnreg split, DESIGN §5); an innocent-looking edit can
push the per-batch state back into local memory or make ptxas serialise the wgmma chain, which costs throughput without
changing a single output bit.  Compiling head_v2_kernel.cu for sm_90a with `-Xptxas=-v` needs nvcc, not a GPU.
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

# spill bytes (stores, loads) of the production instantiations, at most
SPILL_LIMITS = {
    "fp16": (152, 232),    # <false,false>: the benchmarked headline kernel (782 / 958 before the register split)
    "robust": (0, 0),      # <true,false> (624 / 796 before)
}
INST = {"fp16": "_ZN4gfpp9k_head_v2ILb0ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE",
        "robust": "_ZN4gfpp9k_head_v2ILb1ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE"}


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


def _props(report, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\n[^\n]*Used (\d+) registers", report)
    assert m, f"no ptxas report for {mangled}"
    return tuple(int(x) for x in m.groups())


@pytest.mark.parametrize("mode", ["fp16", "robust"])
def test_owner_spills_bounded(ptxas_report, mode):
    _, st, ld, _ = _props(ptxas_report, INST[mode])
    lim_st, lim_ld = SPILL_LIMITS[mode]
    assert st <= lim_st and ld <= lim_ld, f"{mode}: {st} / {ld} bytes of spill stores / loads (limit {lim_st} / {lim_ld})"


@pytest.mark.parametrize("mode", ["fp16", "robust"])
def test_launch_registers_match_split(ptxas_report, mode):
    # the setmaxnreg split assumes the launch allocates 65536 / threads per thread: 128 (3 + 1 warpgroups), 168 (2 + 1)
    _, _, _, regs = _props(ptxas_report, INST[mode])
    assert regs == {"fp16": 128, "robust": 168}[mode]


def test_wgmma_not_serialised(ptxas_report):
    # C7511: "wgmma.mma_async instructions are serialized due to insufficient register resources"
    bad = [l for l in ptxas_report.splitlines() if "C7511" in l and "k_head_v2" in l]
    assert not bad, "\n".join(bad)
