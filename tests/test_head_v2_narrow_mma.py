"""The narrow layers of the row-owner head kernels run as warp-level MMAs on the accumulator registers, checked in the SASS.

Ambient out and colour out (K = 128, N = 3) are chained mma.sync m16n8k16 in the epilogue of the layer that feeds them, with the
A fragments taken from that layer's wgmma accumulators; the sigma row of sigma L2 reads its A fragments back from sigma L1's
stored output with ldmatrix, under colour L0's wgmma (DESIGN §5). Before, each was an N = 16
wgmma group against a resident tile, after an stmatrix epilogue whose only reader it was. These counts pin the instructions of
every k_head_v2 / k_head_v2_train instantiation, so that a narrow product cannot quietly slide back onto the wgmma round trip.
Compiling head_v2_kernel.cu for sm_90a needs nvcc and cuobjdump, not a GPU.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "genefaceplusplus_b200", "csrc", "head_v2_kernel.cu")
CUDA_BIN = os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))

INST = {
    "_ZN4gfpp9k_head_v2ILb0ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": "fp16",
    "_ZN4gfpp9k_head_v2ILb0ELb1EEEvNS_8HeadArgsENS_10HeadV2ArgsE": "fp16",
    "_ZN4gfpp15k_head_v2_trainILb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": "fp16",
    "_ZN4gfpp9k_head_v2ILb1ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": "robust",
    "_ZN4gfpp9k_head_v2ILb1ELb1EEEvNS_8HeadArgsENS_10HeadV2ArgsE": "robust",
    "_ZN4gfpp15k_head_v2_trainILb1EEEvNS_8HeadArgsENS_10HeadV2ArgsE": "robust",
}
# Instructions per kernel.  Each M-half loop is compiled once (#pragma unroll 1), so a narrow product is 8 HMMA (robust ambient
# out: 24, the l*Wh, h*Wl, h*Wh terms).  fp16 HMMA: ambient out 8 + sigma row 8 + colour out 8; robust: 24 + 8 + 8.
# HGMMA and STSM as they were with N = 16 wgmma groups, minus what those groups and the epilogues that fed them took:
#   fp16   HGMMA 67 -> 35: ambient out 8, the sigma row 8, colour out 16 (its loop was unrolled);
#   robust HGMMA 111 -> 63: ambient out 24, the sigma row 8, colour out 16;
#   STSM: colour L0's epilogue (8) in both modes and, fp16, ambient L1's (8): 40 -> 24 and 24 -> 16;
#   LDSM: the sigma row reads sigma L1's stored output back, one ldmatrix per k-block, under colour L0's wgmma.
COUNTS = {
    "fp16": {"HMMA.16816.F32": 24, "HGMMA": 35, "STSM": 24, "LDSM": 8},
    "robust": {"HMMA.16816.F32": 40, "HGMMA": 63, "STSM": 16, "LDSM": 8},
}
# at most, as in test_head_v2_registers.py / test_head_v2_spills.py: (spill stores, spill loads) and the launch registers
SPILL_LIMITS = {
    "_ZN4gfpp9k_head_v2ILb0ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (92, 92),
    "_ZN4gfpp15k_head_v2_trainILb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (116, 116),
    "_ZN4gfpp9k_head_v2ILb1ELb0EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (0, 0),
    "_ZN4gfpp15k_head_v2_trainILb1EEEvNS_8HeadArgsENS_10HeadV2ArgsE": (0, 0),
}
LAUNCH_REGS = {"fp16": 128, "robust": 168}


def _tool(name):
    p = os.path.join(CUDA_BIN, name)
    return p if os.path.exists(p) else shutil.which(name)


@pytest.fixture(scope="module")
def compiled():
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("nvcc / cuobjdump not available")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "v2.o")
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                            "-Xptxas=-v", "-c", SRC, "-o", obj], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        s = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, timeout=300)
        assert s.returncode == 0, s.stderr
    sass, cur = {}, None
    for line in s.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            sass[cur] = []
        elif cur is not None:
            sass[cur].append(line)
    return r.stderr, sass


def _count(lines, op):
    pat = re.compile(r"\s" + re.escape(op) + r"[\s.]")
    return sum(1 for l in lines if pat.search(l))


@pytest.mark.parametrize("mangled", sorted(INST))
def test_narrow_layers_on_mma_sync(compiled, mangled):
    _, sass = compiled
    assert mangled in sass, f"no SASS for {mangled}"
    want = COUNTS[INST[mangled]]
    got = {op: _count(sass[mangled], op) for op in want}
    assert got == want, f"{mangled}: {got}, expected {want}"


@pytest.mark.parametrize("mangled", sorted(SPILL_LIMITS))
def test_owner_registers_and_spills(compiled, mangled):
    report, _ = compiled
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\n[^\n]*Used (\d+) registers", report)
    assert m, f"no ptxas report for {mangled}"
    st, ld, regs = (int(x) for x in m.groups())
    lim_st, lim_ld = SPILL_LIMITS[mangled]
    assert st <= lim_st and ld <= lim_ld, f"{mangled}: {st} / {ld} bytes of spill stores / loads (limit {lim_st} / {lim_ld})"
    assert regs == LAUNCH_REGS[INST[mangled]]
    assert not [l for l in report.splitlines() if "C7511" in l], "wgmma serialised"
