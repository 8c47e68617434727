"""The trainable torso-SR field's C-ABI (gfpp.h section I) and Python guards, without a GPU: every argument is validated before any
CUDA call (a CUDA call on this machine would return GFPP_ERR_CUDA instead of the codes checked here)."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi
from oracle import torso_sr_train as tst
from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR

OK, INVALID, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4
FAKE = 0x10000          # 256-byte aligned, never dereferenced: validation fails or M == 0 returns first
SYMBOLS = ("gfpp_torso_sr_field_workspace_bytes", "gfpp_torso_sr_field_forward", "gfpp_torso_sr_field_backward")
P3 = ctypes.c_void_p * 3


@pytest.fixture(scope="module")
def L():
    from genefaceplusplus_b200 import build
    build.build()
    return _capi.lib()


def _desc(keep, code_dim=8, head_aware=True):
    m = RADNeRFTorsowithSR(tst.golden_hparams("a"))
    d = _capi.TorsoSrDesc()
    d.torso_grid = m._grid_desc(m.torso_embedder, keep)      # host offsets are real; the device pointers are replaced below
    d.torso_grid.embeddings = FAKE
    for i in range(3):
        d.torso_deform_w[i] = d.torso_canon_w[i] = FAKE
        d.ha_w[i] = d.ha_b[i] = FAKE if head_aware else None
    d.torso_code_dim = code_dim
    d.head_aware = int(head_aware)
    d.torso_shrink = 0.8
    return d


def _fwd(L, d, M=128, ws=None, code=FAKE, lm68=FAKE, image=FAKE, wsum=FAKE, out=FAKE):
    ws_bytes = L.gfpp_torso_sr_field_workspace_bytes(0) if ws is None else ws
    return L.gfpp_torso_sr_field_forward(ctypes.byref(d) if d is not None else None, FAKE, M, lm68, code, image, wsum, out, FAKE, FAKE,
                                         FAKE, ws_bytes, None)


def _bwd(L, d, M=128, ws=None, code=FAKE, image=FAKE, wsum=FAKE, grad_code=FAKE, grad_w=True, ha=True, table=FAKE):
    ws_bytes = L.gfpp_torso_sr_field_workspace_bytes(M) if ws is None else ws
    pd, pc, pw, pb = (P3(*([FAKE] * 3)) for _ in range(4))
    return L.gfpp_torso_sr_field_backward(ctypes.byref(d), FAKE, M, FAKE, code, image, wsum, FAKE, FAKE, FAKE,
                                          ctypes.byref(pd) if grad_w else None, ctypes.byref(pc), ctypes.byref(pw) if ha else None,
                                          ctypes.byref(pb) if ha else None, grad_code, table, FAKE, ws_bytes, None)


def test_symbols_and_workspace_sizes(L):
    for n in SYMBOLS:
        assert n in _capi.EXPORTS and hasattr(L, n)
    w0 = L.gfpp_torso_sr_field_workspace_bytes(0)
    assert 0 < w0 < 64_000                                         # the k-major weight and encoder copy and the two folded biases
    assert L.gfpp_torso_sr_field_workspace_bytes(128) > w0         # + one CTA's partial sums
    assert L.gfpp_torso_sr_field_workspace_bytes(10 ** 7) == L.gfpp_torso_sr_field_workspace_bytes(10 ** 8)   # capped CTA count
    assert L.gfpp_torso_sr_field_workspace_bytes(1 << 31) == 0


def test_validation_before_any_cuda_call(L):
    keep = []
    d = _desc(keep)
    assert _fwd(L, None) == INVALID
    assert _fwd(L, d, M=0) == OK and _bwd(L, d, M=0) == OK            # no-op after validation
    assert _fwd(L, d, M=0, out=None) == OK
    assert _fwd(L, d, image=None, wsum=None, M=0) == OK               # the zeros path
    assert _fwd(L, d, out=None) == INVALID                              # null alpha
    assert _fwd(L, d, lm68=None) == INVALID
    assert _fwd(L, d, code=None) == INVALID                             # code must be given iff torso_code_dim > 0
    assert _fwd(L, d, image=None) == INVALID and _fwd(L, d, wsum=None) == INVALID   # image and weights_sum: both or neither
    assert _bwd(L, d, image=None) == INVALID
    assert _fwd(L, d, ws=16) == WORKSPACE
    assert _bwd(L, d, ws=L.gfpp_torso_sr_field_workspace_bytes(0)) == WORKSPACE
    assert _bwd(L, d, grad_w=False) == INVALID
    assert _bwd(L, d, grad_code=None) == INVALID
    assert _bwd(L, d, table=FAKE + 4) == INVALID                        # the table gradient must be 8-byte aligned
    assert _bwd(L, d, ha=False) == INVALID                              # head_aware: grad_ha_* required
    assert _bwd(L, d, ha=False, M=0) == INVALID                         # ... also for M = 0 (validation comes first)
    dn = _desc(keep, head_aware=False)
    assert _fwd(L, dn, M=0, image=None, wsum=None) == OK and _bwd(L, dn, M=0, image=None, wsum=None, ha=False) == OK
    assert _fwd(L, dn, M=0) == INVALID                                  # image / weights_sum are only read with head_aware
    assert _bwd(L, dn, M=0, image=None, wsum=None, ha=True) == INVALID  # grad_ha_* must be NULL without head_aware
    dh = _desc(keep)
    dh.ha_b[1] = None
    assert _fwd(L, dh, M=0) == INVALID                                  # head_aware: the encoder weights are required
    d0 = _desc(keep, code_dim=0)
    assert _fwd(L, d0, code=FAKE) == INVALID and _fwd(L, d0, M=0, code=None) == OK
    assert _fwd(L, _desc(keep, code_dim=11)) == UNSUPPORTED
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


def _cpu_model():
    hp = tst.golden_hparams("a")
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(tst.golden_state(hp), strict=False)
    return m.train()


def test_python_guards_on_a_cpu_model():
    m = _cpu_model()
    x = torch.zeros(4, 2, requires_grad=True)          # would raise NotImplementedError on a GPU model: the CPU check comes first
    with pytest.raises(_capi.GfppNoCpuPath):
        m.forward_torso(x, None, m.torso_individual_codes[torch.tensor([1])], lm68=torch.zeros(1, 136))
    with pytest.raises(_capi.GfppNoCpuPath):
        m.forward_torso(torch.zeros(4, 2), None, None)


def test_gradient_guards_precede_the_kernels(monkeypatch):
    """x, image, weights_sum or lm68 requiring grad raise NotImplementedError in training mode, before anything reaches the device."""
    m = _cpu_model()
    monkeypatch.setattr(m, "_require_cuda", lambda: torch.device("cpu"))
    c = m.torso_individual_codes[torch.tensor([1])]
    x, img, ws, lm = torch.zeros(4, 2), torch.zeros(4, 3), torch.zeros(4, 1), torch.zeros(1, 136)
    for args in ((x.requires_grad_(True), img, ws, lm), (torch.zeros(4, 2), img.clone().requires_grad_(True), ws, lm),
                 (torch.zeros(4, 2), img, ws.clone().requires_grad_(True), lm), (torch.zeros(4, 2), img, ws, lm.clone().requires_grad_(True))):
        with pytest.raises(NotImplementedError, match="not implemented"):
            m.forward_torso(args[0], None, c, args[1], args[2], lm68=args[3])
