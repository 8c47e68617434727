"""The torso pass's C-ABI (gfpp.h section M) and the Python guards of torso_pass(), without a GPU: every argument is validated before
any CUDA call (a CUDA call on this machine would return GFPP_ERR_CUDA instead of the codes checked here), and the new kernels do not
spill."""
import ctypes
import os
import subprocess

import pytest
import torch

from genefaceplusplus_b200 import _capi, build
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR

OK, INVALID, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4
FAKE = 0x10000          # 256-byte aligned, never dereferenced: validation fails first
SYMBOLS = ("gfpp_torso_pass_workspace_bytes", "gfpp_torso_mask", "gfpp_torso_composite_forward", "gfpp_torso_composite_backward")


@pytest.fixture(scope="module")
def L():
    build.build()
    return _capi.lib()


def _mask(L, N=1000, G=64, ws=None, grid=FAKE, xy=FAKE, image=None, wsum=None, image_m=None, wsum_m=None, idx=FAKE, count=FAKE, work=FAKE):
    ws_bytes = L.gfpp_torso_pass_workspace_bytes(N) if ws is None else ws
    return L.gfpp_torso_mask(grid, G, 0.01, xy, N, image, wsum, idx, FAKE, FAKE, image_m, wsum_m, count, work, ws_bytes, None)


def _fwd(L, N=1000, M=10, alpha=FAKE, bg=None, mode=0, image=FAKE, slot=FAKE, out=FAKE):
    return L.gfpp_torso_composite_forward(slot, N, M, alpha, FAKE, image, FAKE, bg, mode, out, FAKE, FAKE, None)


def _bwd(L, N=1000, M=10, idx=FAKE, bg=None, mode=0, grad_alpha=FAKE, alpha=FAKE):
    return L.gfpp_torso_composite_backward(idx, N, M, alpha, FAKE, FAKE, FAKE, bg, mode, None, None, None, grad_alpha, FAKE, None)


def test_symbols_and_workspace_sizes(L):
    for n in SYMBOLS:
        assert n in _capi.EXPORTS and hasattr(L, n)
    assert L.gfpp_torso_pass_workspace_bytes(0) == 0 and L.gfpp_torso_pass_workspace_bytes(1 << 31) == 0
    w1 = L.gfpp_torso_pass_workspace_bytes(1)
    assert w1 == 256 and w1 % 256 == 0
    assert L.gfpp_torso_pass_workspace_bytes((1 << 31) - 1) >= ((1 << 31) // 4096) * 4   # one count per 4096-pixel tile


def test_mask_validation_before_any_cuda_call(L):
    assert _mask(L, grid=None) == INVALID
    assert _mask(L, xy=None) == INVALID
    assert _mask(L, idx=None) == INVALID
    assert _mask(L, count=None) == INVALID
    assert _mask(L, work=None) == INVALID
    assert _mask(L, image=FAKE) == INVALID                                     # the head-aware gathers: all four or none
    assert _mask(L, image=FAKE, wsum=FAKE, image_m=FAKE) == INVALID
    assert _mask(L, N=0, ws=256) == INVALID
    assert _mask(L, N=1 << 31, ws=1 << 20) == UNSUPPORTED
    assert _mask(L, G=1) == UNSUPPORTED and _mask(L, G=4097) == UNSUPPORTED
    assert _mask(L, xy=FAKE + 4) == INVALID                                    # bg_coords must be 8-byte aligned
    assert _mask(L, ws=0) == WORKSPACE
    assert _mask(L, N=10 ** 6, ws=L.gfpp_torso_pass_workspace_bytes(1000)) == WORKSPACE
    assert _mask(L, work=FAKE + 16) == INVALID                                 # workspace must be 256-byte aligned
    assert b"256-byte" in L.gfpp_last_error()


def test_composite_validation_before_any_cuda_call(L):
    assert _fwd(L, slot=None) == INVALID and _fwd(L, out=None) == INVALID and _fwd(L, image=None) == INVALID
    assert _fwd(L, alpha=None) == INVALID                                      # alpha / color needed when M > 0
    assert _fwd(L, N=0, M=0) == INVALID
    assert _fwd(L, N=1 << 31, M=0) == UNSUPPORTED
    assert _fwd(L, N=10, M=11) == INVALID                                      # M > N
    assert _fwd(L, mode=3, bg=FAKE) == INVALID
    assert _fwd(L, mode=1, bg=None) == INVALID and _fwd(L, mode=2, bg=None) == INVALID
    assert _fwd(L, mode=0, bg=FAKE) == INVALID
    assert _bwd(L, idx=None) == INVALID and _bwd(L, grad_alpha=None) == INVALID and _bwd(L, alpha=None) == INVALID
    assert _bwd(L, N=10, M=11) == INVALID and _bwd(L, mode=1) == INVALID and _bwd(L, mode=5, bg=FAKE) == INVALID
    assert _bwd(L, N=0, M=0) == INVALID
    assert _bwd(L, M=0, idx=None, grad_alpha=None, alpha=None) == OK          # nothing to do: no device access
    assert L.gfpp_last_launch_count() == 0


def test_new_kernels_do_not_spill():
    cu = os.path.join(build.CSRC, "torso_pass_kernels.cu")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas=-v", "-c", cu, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    entries = [ln for ln in r.stderr.splitlines() if "Compiling entry function" in ln and "torso_" in ln]
    assert len(entries) == 5, r.stderr
    stacks = [ln for ln in r.stderr.splitlines() if "spill stores" in ln]
    assert len(stacks) == 5 and all("0 bytes spill stores, 0 bytes spill loads" in ln for ln in stacks), stacks


def _torso_model():
    sc = scn.Scene(H=16, W=16, T=2, torso=True)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    return m.train()


def _sr_model():
    from oracle import torso_sr_train as tst
    hp = tst.golden_hparams("b")
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(tst.golden_state(hp), strict=False)
    return m.train()


def _args(N=256):
    return dict(image=torch.rand(N, 3), weights_sum=torch.rand(N), bg_coords=torch.rand(N, 2) * 2 - 1)


def test_cpu_model_raises_no_cpu_path():
    m = _torso_model()
    a = _args()
    with pytest.raises(_capi.GfppNoCpuPath):
        m.torso_pass(a["image"], a["weights_sum"], a["bg_coords"], torch.zeros(1, 6), m.torso_individual_codes[torch.tensor([1])])
    with pytest.raises(_capi.GfppNoCpuPath):      # before the gradient guard
        m.torso_pass(a["image"].requires_grad_(True), a["weights_sum"], a["bg_coords"], torch.zeros(1, 6), m.torso_individual_codes[0:1])
    s = _sr_model()
    with pytest.raises(_capi.GfppNoCpuPath):
        s.torso_pass(a["image"], a["weights_sum"], a["bg_coords"], None, s.torso_individual_codes[0:1], lm68=torch.zeros(136))


@pytest.mark.parametrize("cls", ["torso", "sr"])
def test_guards_precede_the_kernels(monkeypatch, cls):
    """Inputs that require grad raise NotImplementedError and shape mismatches ValueError, before anything reaches the device."""
    m = _torso_model() if cls == "torso" else _sr_model()
    monkeypatch.setattr(m, "_require_cuda", lambda: torch.device("cpu"))
    monkeypatch.setattr(_capi, "lib", lambda: pytest.fail("the library was reached"))
    c = m.torso_individual_codes[torch.tensor([1])]
    cond = dict(poses=torch.zeros(1, 6), lm68=None) if cls == "torso" else dict(poses=None, lm68=torch.zeros(1, 136))
    N = 256

    def call(**kw):
        a = {**_args(N), **cond, "c": c, "bg_color": None, **kw}
        return m.torso_pass(a["image"], a["weights_sum"], a["bg_coords"], a["poses"], a["c"], bg_color=a["bg_color"], lm68=a["lm68"])

    for k, shape in (("image", (N, 3)), ("weights_sum", (N,)), ("bg_coords", (N, 2)), ("bg_color", (3,))):
        with pytest.raises(NotImplementedError):
            call(**{k: torch.rand(*shape, requires_grad=True)})
    grad_cond = "poses" if cls == "torso" else "lm68"
    with pytest.raises(NotImplementedError):
        call(**{grad_cond: torch.zeros(*cond[grad_cond].shape, requires_grad=True)})
    with pytest.raises(ValueError):
        call(image=torch.rand(N - 1, 3))
    with pytest.raises(ValueError):
        call(weights_sum=torch.rand(N + 1))
    with pytest.raises(ValueError):
        call(bg_coords=torch.rand(N, 3))
    with pytest.raises(ValueError):
        call(bg_color=torch.rand(4))
    with pytest.raises(ValueError):
        call(bg_color=torch.rand(N - 1, 3))
    with pytest.raises(ValueError):
        call(c=None)
    with pytest.raises(ValueError):
        call(c=torch.zeros(1, 3))
    if cls == "torso":
        with pytest.raises(ValueError):
            call(poses=torch.zeros(1, 5))
    else:
        with pytest.raises(ValueError):
            call(lm68=None)
        with pytest.raises(ValueError):
            call(lm68=torch.zeros(68))
