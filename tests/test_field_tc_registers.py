"""The tensor-core training field's kernels (csrc/field_train_tc_kernel.cu) compiled for sm_90a with -Xptxas=-v report no register
spills.  CPU only: nvcc cross-compiles."""
import os
import re
import subprocess
import tempfile

from genefaceplusplus_b200 import build

KERNELS = ("k_field_tc_relayout", "k_field_tc_fwd", "k_field_tc_bwd")


def test_no_spills():
    with tempfile.TemporaryDirectory() as td:
        cmd = [build.NVCC, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "field_train_tc_kernel.cu"), "-o", os.path.join(td, "k.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rep, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            rep.setdefault(cur, {})["spill"] = (int(m.group(2)), int(m.group(3)))
            rep[cur]["stack"] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            rep[cur]["regs"] = int(m.group(1))
    found = {n: v for n in KERNELS for k, v in rep.items() if re.search(rf"\d{n}E", k)}
    assert sorted(found) == sorted(KERNELS), rep
    for k, v in found.items():
        print(f"{k}: {v['regs']} registers, {v['stack']} bytes stack, spills {v['spill']}")
        assert v["spill"] == (0, 0), (k, v)
