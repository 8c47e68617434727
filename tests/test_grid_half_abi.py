"""C-ABI section (L), the grid encoder on half tables, without a GPU: argument validation before any CUDA call, the shims' dtype
dispatch refusing mixed buffers, and the half checker against its own fp32 evaluation (one binary16 ulp per rounding site)."""
import ctypes

import numpy as np
import pytest
import torch

from checkers import grid_half as gh
from genefaceplusplus_b200 import _capi, backend_shims

P = ctypes.c_void_p
OFF3 = (ctypes.c_int32 * 17)(*[i * 64 for i in range(17)])      # 16 levels of 64 entries


def _fwd(L, *a):
    return L.gfpp_grid_encode_forward_half(*a)


def test_exports_are_declared_and_loaded():
    L = _capi.lib()
    for n in ("gfpp_grid_encode_forward_half", "gfpp_grid_encode_backward_half"):
        assert n in _capi.EXPORTS and hasattr(L, n)


def test_forward_validates_before_any_cuda_call():
    L = _capi.lib()
    ok = (P(64), P(64), OFF3, P(64), 0, 3, 2, 16, 0.5, 16, None, 1, 0, 0, None)
    assert _fwd(L, *ok) == 0                          # B == 0 passes validation and returns before touching the device
    for i in (0, 1, 2, 3):                            # inputs, embeddings, offsets, outputs
        a = list(ok); a[i] = None
        assert _fwd(L, *a) == -1 and b"null" in L.gfpp_last_error()
    for i, v, word in ((6, 4, b"C == 2"), (5, 4, b"D must be"), (5, 1, b"D must be"), (7, 17, b"L <= 16"), (7, 0, b"L <= 16")):
        a = list(ok); a[i] = v
        assert _fwd(L, *a) == -4 and word in L.gfpp_last_error(), (i, v)
    a = list(ok); a[1] = P(66)                        # a half2 table must be 4-byte aligned
    assert _fwd(L, *a) == -1 and b"aligned" in L.gfpp_last_error()
    a = list(ok); a[10] = P(70)
    assert _fwd(L, *a) == -1 and b"aligned" in L.gfpp_last_error()
    empty = (ctypes.c_int32 * 17)(*([0] * 17))         # empty levels
    a = list(ok); a[2] = empty
    assert _fwd(L, *a) == -4


def test_backward_validates_before_any_cuda_call():
    L = _capi.lib()
    ok = [P(64), P(64), P(64), OFF3, P(64), 0, 3, 2, 16, 0.5, 16, P(64), P(64), 1, 0, 0, None]
    assert L.gfpp_grid_encode_backward_half(*ok) == 0                                  # B == 0: nothing launched
    for i in (0, 1, 3, 4):                                                             # grad, inputs, offsets, grad_embeddings
        a = list(ok); a[i] = None
        assert L.gfpp_grid_encode_backward_half(*a) == -1 and b"null" in L.gfpp_last_error()
    a = list(ok); a[12] = None                                                         # dy_dx without grad_inputs
    assert L.gfpp_grid_encode_backward_half(*a) == -1 and b"together" in L.gfpp_last_error()
    a = list(ok); a[11] = None                                                         # grad_inputs without dy_dx
    assert L.gfpp_grid_encode_backward_half(*a) == -1 and b"together" in L.gfpp_last_error()
    for i, v in ((7, 1), (7, 8), (6, 4), (8, 17)):
        a = list(ok); a[i] = v
        assert L.gfpp_grid_encode_backward_half(*a) == -4, (i, v)
    a = list(ok); a[4] = P(66)
    assert L.gfpp_grid_encode_backward_half(*a) == -1 and b"aligned" in L.gfpp_last_error()


def test_shims_refuse_mixed_dtypes():
    """A half table with fp32 outputs / dy_dx, or a half backward with any fp32 gradient buffer, raises RuntimeError like the
    reference's data_ptr<at::Half>() -- before any pointer reaches the library."""
    ge = backend_shims.make_modules()["_gridencoder"]
    B, D, Lv = 4, 3, 16
    off = torch.arange(17, dtype=torch.int32) * 64
    x = torch.rand(B, D)
    emb_h, emb_f = torch.zeros(16 * 64, 2, dtype=torch.half), torch.zeros(16 * 64, 2)
    out_h, out_f = torch.empty(Lv, B, 2, dtype=torch.half), torch.empty(Lv, B, 2)
    dd_h, dd_f = torch.empty(B, Lv * D * 2, dtype=torch.half), torch.empty(B, Lv * D * 2)
    with pytest.raises(RuntimeError, match="outputs must be float16"):
        ge.grid_encode_forward(x, emb_h, off, out_f, B, D, 2, Lv, 0.5, 16, None, 1, False, 0)
    with pytest.raises(RuntimeError, match="dy_dx must be float16"):
        ge.grid_encode_forward(x, emb_h, off, out_h, B, D, 2, Lv, 0.5, 16, dd_f, 1, False, 0)
    g_h, g_f = torch.zeros(Lv, B, 2, dtype=torch.half), torch.zeros(Lv, B, 2)
    ge_h, ge_f = torch.zeros_like(emb_h), torch.zeros_like(emb_f)
    gi_h, gi_f = torch.zeros(B, D, dtype=torch.half), torch.zeros(B, D)
    for grad, emb, gemb, dd, gi, name in ((g_h, emb_h, ge_f, None, None, "grad_embeddings"), (g_h, emb_f, ge_h, None, None, "embeddings"),
                                          (g_f, emb_h, ge_h, None, None, "grad must"), (g_h, emb_h, ge_h, dd_h, gi_f, "grad_inputs"),
                                          (g_h, emb_h, ge_h, dd_f, gi_h, "dy_dx")):
        with pytest.raises(RuntimeError, match=name):
            ge.grid_encode_backward(grad, x, emb, off, gemb, B, D, 2, Lv, 0.5, 16, dd, gi, 1, False, 0)
    with pytest.raises(RuntimeError, match="fp32 or fp16"):
        ge.grid_encode_forward(x, emb_f.double(), off, out_f, B, D, 2, Lv, 0.5, 16, None, 1, False, 0)


def _grid(D, gridtype, seed):
    """A small grid with a dense low part and capped (hashed when gridtype == 0) fine levels: 8 levels, base 4, x1.6 per level."""
    L, H, pls, cap = 8, 4, 1.6, 2 ** 9
    offs, o = [0], 0
    for l in range(L):
        res = int(np.ceil(H * pls ** l))
        n = min(cap, (res + 1) ** D)
        n = int(np.ceil(n / 8) * 8)
        o += n
        offs.append(o)
    g = torch.Generator().manual_seed(seed)
    emb = ((torch.rand(o, 2, generator=g) - 0.5) * 2).half()
    return emb, torch.tensor(offs, dtype=torch.int32), float(np.log2(pls)), H


VARIANTS = [(D, gt, it, al) for D in (2, 3) for gt in (0, 1) for it in (0, 1) for al in (False, True)]


@pytest.mark.parametrize("D,gridtype,interp,align", VARIANTS)
def test_checker_half_within_one_ulp_per_rounding_site_of_fp32(D, gridtype, interp, align):
    emb, off, S, H = _grid(D, gridtype, 7 + D)
    g = torch.Generator().manual_seed(11)
    B = 500
    x = torch.rand(B, D, generator=g)
    x[:3] = torch.tensor([1.0, 0.0, 0.5])[:D]           # faces of the unit cube
    x[3, 0] = 1.0001                                    # out of range: zeros
    L = off.numel() - 1
    kw = dict(gridtype=gridtype, align_corners=align, interp=interp, dy_dx=True)
    oh, dh = gh.forward(x, emb, off, S, H, rnd=True, **kw)
    of, df = gh.forward(x, emb, off, S, H, rnd=False, **kw)
    assert torch.equal(oh, gh.forward(x, emb, off, S, H, rnd=True, **kw)[0])
    assert torch.equal(oh.half().float(), oh) and torch.equal(dh.half().float(), dh)     # every result is a binary16 value
    assert (oh[:, 3] == 0).all() and (dh[3] == 0).all()
    # outputs: 2 sites per corner (term, sum); every partial value is bounded by the sum of |w g|
    mag, _ = gh.forward(x, emb.float().abs(), off, S, H, rnd=False, **kw)
    tol = 2 * 2 ** D * gh.ulp16(mag.numpy())
    assert (np.abs((oh - of).numpy()) <= tol).all()
    # dy_dx: 3 sites per term (difference, term, sum); partial values bounded by scale * max|deriv| * 2 max|g| per level
    scale = np.array([np.float32(np.exp2(np.float32(l * S)) * H - 1) for l in range(L)])
    amax = np.array([emb[off[l]:off[l + 1]].float().abs().max().item() for l in range(L)])
    bound = scale * (1.5 if interp else 1.0) * 2 * amax
    tol = (3 * 2 ** (D - 1) * gh.ulp16(bound))[None, :, None, None]
    assert (np.abs((dh - df).numpy()) <= tol).all()
    # input gradient: 2 sites per (level, channel), partials bounded by sum |grad dy_dx|
    grad = (torch.randn(L, B, 2, generator=g) * 0.1).half().float()
    gih = gh.input_grad(grad, dh, rnd=True)
    gif = gh.input_grad(grad, dh, rnd=False)
    gmag = gh.input_grad(grad.abs(), dh.abs(), rnd=False)
    assert (np.abs((gih - gif).numpy()) <= 2 * 2 * L * gh.ulp16(gmag.numpy())).all()
    # table gradient: one rounding per added term, each within half an ulp of its fp32 value
    sh, ah, kh = gh.table_grad(grad, x, off, emb.shape[0], S, H, gridtype=gridtype, align_corners=align, interp=interp, rnd=True)
    sf, af, kf = gh.table_grad(grad, x, off, emb.shape[0], S, H, gridtype=gridtype, align_corners=align, interp=interp, rnd=False)
    assert torch.equal(kh, kf) and int(kh.sum()) == (B - 1) * L * 2 ** D
    assert ((sh - sf).abs().numpy() <= kh[:, None].numpy() * gh.ulp16(af.numpy()) + 1e-30).all()


def test_checker_binary16_rounding_matches_torch():
    """The checker's float -> binary16 conversion (round to nearest even, subnormals, overflow to inf) against torch's."""
    g = torch.Generator().manual_seed(3)
    n = 20_000
    x = torch.randn(n, generator=g) * torch.exp2(torch.empty(n).uniform_(-30, 17, generator=g))
    x[:6] = torch.tensor([65504.0, 65519.99, 65520.0, 2.0 ** -25, 3 * 2.0 ** -26, -2.0 ** -24])
    got = torch.tensor([gh.round_half(float(v)) for v in x])
    assert torch.equal(got, x.half().float())
