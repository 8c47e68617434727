"""The torso-SR training kernels (csrc/torso_sr_train_kernel.cu and the point mode of k_torso_sr, csrc/torso_sr_points_kernel.cu)
compiled for sm_90a with -Xptxas=-v report no register spills.  CPU only: nvcc cross-compiles."""
import os
import re
import subprocess
import tempfile

import pytest

from genefaceplusplus_b200 import build

KERNELS = ("k_torso_sr_field_relayout", "k_torso_sr_field_bwd", "k_torso_sr_field_reduce", "k_torso_sr_points")


def _ptxas_report(src):
    with tempfile.TemporaryDirectory() as td:
        cmd = [build.NVCC, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, src), "-o", os.path.join(td, "k.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
    return out


@pytest.mark.parametrize("src", ["torso_sr_train_kernel.cu", "torso_sr_points_kernel.cu"])
def test_no_spills(src):
    rep = _ptxas_report(src)
    found = {k: v for k, v in rep.items() if any(n in k for n in KERNELS)}
    assert found, rep
    for k, (st, ld) in found.items():
        print(f"{k}: {st} bytes spill stores, {ld} bytes spill loads")
        assert st == 0 and ld == 0, (k, st, ld)
