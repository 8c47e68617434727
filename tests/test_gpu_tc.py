"""wgmma plumbing self-test: one 128 x N x K GEMM through the exact tile layouts / descriptors / accumulator fragment read-back of
the tensor-core MLP, against a float64 reference with operands rounded the way the kernel rounds them."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi

pytestmark = pytest.mark.gpu

SHAPES = [(128, 64, 0), (128, 96, 0), (128, 128, 0), (144, 128, 0), (16, 128, 0), (128, 144, 1), (128, 80, 1)]


def _round(x, precision):
    if precision == 1:
        return x.half().double()
    return x.bfloat16().double()


@pytest.mark.parametrize("precision", [1, 3, 2], ids=["fp16", "bf16", "bf16x3"])
@pytest.mark.parametrize("N,K,k16", SHAPES)
def test_tc_gemm(N, K, k16, precision):
    g = torch.Generator().manual_seed(N * 1000 + K)
    A = torch.randn(128, K, generator=g)
    W = torch.randn(N, K, generator=g) / (K ** 0.5)
    Ad, Wd = A.cuda(), W.cuda()
    out = torch.full((128, N), float("nan"), device="cuda")
    scratch = torch.empty(6 * 18432, dtype=torch.uint8, device="cuda")
    rc = _capi.lib().gfpp_tc_selftest(Ad.data_ptr(), Wd.data_ptr(), N, K, k16, precision, scratch.data_ptr(), out.data_ptr(), _capi.stream_ptr())
    _capi.check(rc, "tc_selftest")
    torch.cuda.synchronize()
    exact = A.double() @ W.double().t()
    if precision == 2:
        ah, wh = _round(A, 2), _round(W, 2)
        al, wl = _round(A - ah.float(), 2), _round(W - wh.float(), 2)
        ref = ah @ wh.t() + ah @ wl.t() + al @ wh.t()
        tol_exact = 2e-4
    else:
        ref = _round(A, precision) @ _round(W, precision).t()
        tol_exact = 5e-3 if precision == 1 else 4e-2
    got = out.cpu().double()
    assert torch.isfinite(got).all()
    err_model = (got - ref).abs().max().item()
    err_exact = (got - exact).abs().max().item()
    print(f"N={N} K={K} k16={k16} prec={precision}: |got - rounded-operand ref| = {err_model:.2e}, |got - exact| = {err_exact:.2e}")
    assert err_model < 2e-5 * max(1.0, exact.abs().max().item()), "layout / descriptor error (not a rounding effect)"
    assert err_exact < tol_exact * max(1.0, exact.abs().max().item())
