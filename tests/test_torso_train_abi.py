"""The trainable torso field's C-ABI (gfpp.h section H) and Python guards, without a GPU: every argument is validated before any CUDA
call (a CUDA call on this machine would return GFPP_ERR_CUDA instead of the codes checked here)."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRFTorso

OK, INVALID, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4
FAKE = 0x10000          # 256-byte aligned, never dereferenced: validation fails or M == 0 returns first
SYMBOLS = ("gfpp_torso_field_workspace_bytes", "gfpp_torso_field_forward", "gfpp_torso_field_backward")


@pytest.fixture(scope="module")
def L():
    from genefaceplusplus_b200 import build
    build.build()
    return _capi.lib()


def _desc(keep, code_dim=8):
    m = RADNeRFTorso(may_hparams())
    d = _capi.ModelDesc()
    m._fill_desc(d, keep)          # host offsets are real; the device pointers are replaced below
    d.torso_grid.embeddings = FAKE
    for i in range(3):
        d.torso_deform_w[i] = FAKE
        d.torso_canon_w[i] = FAKE
    d.torso_code_dim = code_dim
    return d


def _fwd(L, d, M=128, ws=None, code=FAKE, pose=FAKE, out=FAKE):
    ws_bytes = L.gfpp_torso_field_workspace_bytes(0) if ws is None else ws
    return L.gfpp_torso_field_forward(ctypes.byref(d) if d is not None else None, FAKE, M, pose, code, out, FAKE, FAKE, FAKE, ws_bytes, None)


def _bwd(L, d, M=128, ws=None, code=FAKE, grad_code=FAKE, grad_w=True, table=FAKE):
    ws_bytes = L.gfpp_torso_field_workspace_bytes(M) if ws is None else ws
    pd = (ctypes.c_void_p * 3)(*([FAKE] * 3))
    pc = (ctypes.c_void_p * 3)(*([FAKE] * 3))
    return L.gfpp_torso_field_backward(ctypes.byref(d), FAKE, M, FAKE, code, FAKE, FAKE, FAKE, ctypes.byref(pd) if grad_w else None,
                                       ctypes.byref(pc), grad_code, table, FAKE, ws_bytes, None)


def test_symbols_and_workspace_sizes(L):
    for n in SYMBOLS:
        assert n in _capi.EXPORTS and hasattr(L, n)
    w0 = L.gfpp_torso_field_workspace_bytes(0)
    assert 0 < w0 < 64_000                                     # the k-major weight copy and the two folded biases
    assert L.gfpp_torso_field_workspace_bytes(128) > w0        # + one CTA's partial sums
    assert L.gfpp_torso_field_workspace_bytes(10 ** 7) == L.gfpp_torso_field_workspace_bytes(10 ** 8)   # capped CTA count
    assert L.gfpp_torso_field_workspace_bytes(1 << 31) == 0


def test_validation_before_any_cuda_call(L):
    keep = []
    d = _desc(keep)
    assert _fwd(L, None) == INVALID
    assert _fwd(L, d, M=0) == OK and _bwd(L, d, M=0) == OK        # no-op after validation
    assert _fwd(L, d, M=0, out=None) == OK
    assert _fwd(L, d, out=None) == INVALID                          # null alpha
    assert _fwd(L, d, pose=None) == INVALID
    assert _fwd(L, d, code=None) == INVALID                         # code must be given iff torso_code_dim > 0
    assert _fwd(L, d, ws=16) == WORKSPACE
    assert _bwd(L, d, ws=L.gfpp_torso_field_workspace_bytes(0)) == WORKSPACE
    assert _bwd(L, d, grad_w=False) == INVALID
    assert _bwd(L, d, grad_code=None) == INVALID
    assert _bwd(L, d, table=FAKE + 4) == INVALID                    # the table gradient must be 8-byte aligned
    d0 = _desc(keep, code_dim=0)
    assert _fwd(L, d0, code=FAKE) == INVALID and _fwd(L, d0, M=0, code=None) == OK
    assert _fwd(L, _desc(keep, code_dim=11)) == UNSUPPORTED         # the code dimensions the inference query accepts: <= 10
    d2 = _desc(keep)
    d2.torso_grid.num_levels = 8
    assert _fwd(L, d2) == UNSUPPORTED
    d3 = _desc(keep)
    d3.torso_grid.input_dim = 3
    assert _fwd(L, d3) == UNSUPPORTED
    d4 = _desc(keep)
    d4.torso_canon_w[1] = None
    assert _fwd(L, d4) == INVALID and _bwd(L, d4) == INVALID
    d5 = _desc(keep)
    d5.torso_grid.embeddings = FAKE + 4
    assert _fwd(L, d5) == INVALID
    assert _fwd(L, d, M=1 << 31) == UNSUPPORTED


def test_python_guards_on_a_cpu_model():
    sc = scn.Scene(H=16, W=16, T=2, torso=True)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.train()
    x = torch.zeros(4, 2, requires_grad=True)          # would raise NotImplementedError on a GPU model: the CPU check comes first
    with pytest.raises(_capi.GfppNoCpuPath):
        m.forward_torso(x, torch.zeros(1, 6), m.torso_individual_codes[torch.tensor([1])])
    with pytest.raises(_capi.GfppNoCpuPath):
        m.forward_torso(torch.zeros(4, 2), torch.zeros(1, 6), None)
    m.eval()
    with pytest.raises(_capi.GfppNoCpuPath):
        m.forward_torso(torch.zeros(4, 2), torch.zeros(1, 6), m.torso_individual_codes[0:1])


def test_gradient_guards_precede_the_kernels(monkeypatch):
    """x or poses requiring grad raise NotImplementedError in training mode, before anything reaches the device."""
    sc = scn.Scene(H=16, W=16, T=2, torso=True)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.train()
    monkeypatch.setattr(m, "_require_cuda", lambda: torch.device("cpu"))
    c = m.torso_individual_codes[torch.tensor([1])]
    with pytest.raises(NotImplementedError, match="positions or the head pose"):
        m.forward_torso(torch.zeros(4, 2, requires_grad=True), torch.zeros(1, 6), c)
    with pytest.raises(NotImplementedError, match="positions or the head pose"):
        m.forward_torso(torch.zeros(4, 2), torch.zeros(1, 6, requires_grad=True), c)
