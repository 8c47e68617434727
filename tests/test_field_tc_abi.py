"""The tensor-core training field's C-ABI (gfpp.h section J) and RADNeRF.train_precision, without a GPU: every argument is validated
before any CUDA call (a CUDA call on this machine would return GFPP_ERR_CUDA instead of the codes checked here)."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF

OK, INVALID, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4
FAKE = 0x10000          # 256-byte aligned, never dereferenced: validation fails or M == 0 returns first
IMAGES = 344064 + 1024  # the fp16 weight images and the two folded biases (FieldTcImg)


@pytest.fixture(scope="module")
def L():
    from genefaceplusplus_b200 import build
    build.build()
    return _capi.lib()


def _desc(keep, amb_dim=3, ind_dim=4):
    m = RADNeRF(may_hparams(ambient_coord_dim=amb_dim))
    d = _capi.ModelDesc()
    m._fill_desc(d, keep)          # host offsets are real; the device pointers are replaced below
    d.position_grid.embeddings = FAKE
    d.ambient_grid.embeddings = FAKE
    for i in range(3):
        d.ambient_w[i] = FAKE
        d.sigma_w[i] = FAKE
    for i in range(2):
        d.color_w[i] = FAKE
    d.ind_dim = ind_dim
    d.individual_code = FAKE if ind_dim else None
    return d


def _fwd(L, d, M=128, ws=None, ws_ptr=FAKE):
    ws_bytes = L.gfpp_field_tc_workspace_bytes(0) if ws is None else ws
    return L.gfpp_field_tc_forward(ctypes.byref(d) if d is not None else None, FAKE, FAKE, M, FAKE, FAKE, FAKE, FAKE, ws_ptr, ws_bytes, None)


def _bwd(L, d, M=128, ws=None, grad_w=True, tab=FAKE):
    ws_bytes = L.gfpp_field_tc_workspace_bytes(M) if ws is None else ws
    ptrs = (ctypes.c_void_p * 8)(*([FAKE] * 8))
    return L.gfpp_field_tc_backward(ctypes.byref(d), FAKE, FAKE, M, FAKE, FAKE, FAKE, FAKE, ctypes.byref(ptrs) if grad_w else None, FAKE, FAKE,
                                    tab, FAKE, FAKE, ws_bytes, None)


def test_symbols_and_workspace_sizes(L):
    for n in ("gfpp_field_tc_workspace_bytes", "gfpp_field_tc_forward", "gfpp_field_tc_backward"):
        assert n in _capi.EXPORTS and hasattr(L, n)
    sizes = [L.gfpp_field_tc_workspace_bytes(M) for M in (0, 1, 128, 129, 5000, 132 * 128, 10 ** 7, 10 ** 8)]
    assert sizes[0] == IMAGES
    assert all(a <= b for a, b in zip(sizes, sizes[1:])) and sizes[1] > sizes[0] and sizes[3] > sizes[2]
    assert sizes[1] == sizes[2]                               # one 128-point tile, one CTA's partial sums
    assert sizes[-1] == sizes[-2] == sizes[-3]                # capped CTA count
    assert L.gfpp_field_tc_workspace_bytes(1 << 30) == 0


def test_validation_before_any_cuda_call(L):
    keep = []
    assert _fwd(L, None) == INVALID
    for amb_dim in (2, 3):
        for ind_dim in (0, 4, 16):
            d = _desc(keep, amb_dim, ind_dim)
            assert _fwd(L, d, M=0) == OK and _bwd(L, d, M=0) == OK       # M == 0: a no-op
            assert _fwd(L, d, ws=IMAGES - 1) == WORKSPACE
            assert _bwd(L, d, ws=L.gfpp_field_tc_workspace_bytes(128) - 1) == WORKSPACE
    d = _desc(keep)
    assert _fwd(L, d, ws_ptr=FAKE + 64) == INVALID            # workspace must be 256-byte aligned
    assert _fwd(L, d, ws_ptr=None) == INVALID
    assert _bwd(L, d, tab=FAKE + 4) == INVALID                # table gradients must be 8-byte aligned
    assert _bwd(L, d, grad_w=False) == INVALID
    d.sigma_w[1] = None
    assert _fwd(L, d) == INVALID and _bwd(L, d) == INVALID
    d = _desc(keep)
    d.color_w[0] = FAKE + 4                                   # weights must be 16-byte aligned
    assert _fwd(L, d) == INVALID
    d = _desc(keep)
    d.mlp_precision = 1                                       # names the inference arithmetic; the training switch is the entry point
    assert _fwd(L, d) == UNSUPPORTED and _bwd(L, d) == UNSUPPORTED
    assert _fwd(L, _desc(keep, ind_dim=3)) == UNSUPPORTED
    d = _desc(keep)
    d.individual_code = None                                  # ind_dim 4 without a code
    assert _fwd(L, d) == INVALID
    d = _desc(keep)
    d.cond_dim = 32
    assert _fwd(L, d) == UNSUPPORTED
    d = _desc(keep)
    d.position_grid.input_dim = 2
    assert _fwd(L, d) == UNSUPPORTED
    d = _desc(keep)
    d.ambient_grid.num_levels = 8
    assert _bwd(L, d) == UNSUPPORTED
    assert _fwd(L, _desc(keep), M=1 << 30) == UNSUPPORTED
    assert b"field_tc_forward" in L.gfpp_last_error()


def test_train_precision_values():
    assert RADNeRF(may_hparams()).train_precision == "fp32"
    hp = may_hparams()
    hp["gfpp_train_precision"] = "fp16"
    assert RADNeRF(hp).train_precision == "fp16"
    m = RADNeRF(may_hparams())
    m.train_precision = "bogus"
    with pytest.raises(ValueError, match="train_precision"):
        m.forward(torch.zeros(4, 3), torch.zeros(4, 3), torch.zeros(1, 64), None)


def test_cpu_model_has_no_cpu_path():
    sc = scn.Scene(H=8, W=8, T=2, torso=False)
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.train_precision = "fp16"
    m.train()
    fi = sc.frame_inputs(0)
    with pytest.raises(_capi.GfppNoCpuPath):
        m.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], **sc.hparams)
    with pytest.raises(_capi.GfppNoCpuPath):
        m.forward(torch.zeros(4, 3), torch.zeros(4, 3), torch.zeros(1, 64), m.individual_embeddings[0])
