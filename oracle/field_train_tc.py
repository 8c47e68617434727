"""oracle/field_train_tc.py -- TEST INFRASTRUCTURE (CPU checker; never imported by the product path).

The rounding contract of libgfpp's tensor-core training field (gfpp.h section J, csrc/field_train_tc_kernel.cu) in code:
oracle/field_train.field_forward with `x.half()` at exactly the sites the kernels round, fp32 (or the weights' dtype) everywhere else.

  * forward: the operands of the six wide products -- activations (grid features, SH, hidden layers) and weights -- are rounded to
    fp16; the conditioning vector and the individual code are the same for every point, so their columns of ambient_net.0 /
    color_net.0 are a bias computed without rounding; the narrow layers (ambient_net.2, row 0 of sigma_net.2, color_net.1) read the
    unrounded activations, so nothing rounded to 16 bits enters tanh, exp or the sigmoid directly;
  * backward of a wide product: the output gradient dY is multiplied by a power of two, rounded to fp16 and the products
    dX = dY W, dW = dY^T X (rounded W and X) are scaled back; the folded columns' gradients are column sums of the same rounded dY.
    The power of two is the kernels' block_scale: one per block of TILE (= FIELD_TC_TP = 128) consecutive points, over all of that
    block's columns, bringing the block's largest magnitude to [256, 512) (exponent clamped to +-126); 1 for a block that is all
    zero or whose largest magnitude is infinite.  NaNs do not count towards the largest magnitude (fmaxf drops them).  Rows past
    the call's last point are zero, so they never change the last block's scale.  A block whose points are many binades fainter
    than another's keeps its own 11 bits: a faint tile of a training step is not flushed by a loud one.
  * backward of a narrow layer: fp32, with the layer's input as the fp16 value the kernels keep in shared memory for dW.

    sigma, color, ambient_pos = field_forward(params, hparams, xyzs, dirs, cond_feat, individual_code, rounding=True, trace=None)

trace: an optional dict that receives, under "relu_pre", the pre-activations [N,128] of the five ReLUs (ambient 2, sigma 2, colour 1)
as this arithmetic computes them, as oracle/field_train.field_forward records its own.  With rounding=False every layer is
torch.nn.functional.linear on the concatenated input, as in oracle/field_train.py, bit for bit.
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch.autograd import Function

from . import field_train as ft
from . import ops


def _r16(x):
    return x.half().to(x.dtype)


TILE = 128   # FIELD_TC_TP: the points of one block of the scale rule


def block_exponents(g, rows=None):
    """The exponent k of block_scale for each block of `rows` (default TILE) consecutive rows of g [n, C]: 2^k brings the block's
    largest magnitude (NaNs ignored) to [256, 512), k in [-126, 126]; 0 where that magnitude is 0 or infinite."""
    n = g.shape[0]
    rows = min(TILE if rows is None else rows, max(n, 1))   # a block past the call's end holds the call
    nb = -(-max(n, 1) // rows)
    a = g.detach().abs()
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
    m = F.pad(a.reshape(n, -1), (0, 0, 0, nb * rows - n)).reshape(nb, -1).amax(1)
    _, e = torch.frexp(m)                        # m = f 2^e, f in [0.5, 1): the largest magnitude's binade is 2^(e-1)
    k = (9 - e).clamp(-126, 126)
    return torch.where((m > 0) & torch.isfinite(m), k, torch.zeros_like(k))


def _r16_scaled(g):
    """g [n, C] rounded to fp16 under block_scale's power of two per TILE rows, and scaled back."""
    rows = min(TILE, max(g.shape[0], 1))
    k = block_exponents(g, rows).repeat_interleave(rows)[:g.shape[0]].reshape(-1, *([1] * (g.dim() - 1)))
    return torch.ldexp(_r16(torch.ldexp(g, k)), -k)


class _WideTC(Function):
    """y = r16(x) r16(w)^T; dX = r16s(dY) r16(w), dW = r16s(dY)^T r16(x)."""

    @staticmethod
    def forward(ctx, x, w):
        xr, wr = _r16(x), _r16(w)
        ctx.save_for_backward(xr, wr)
        return F.linear(xr, wr)

    @staticmethod
    def backward(ctx, g):
        xr, wr = ctx.saved_tensors
        gr = _r16_scaled(g)
        return gr @ wr, gr.t() @ xr


class _FoldTC(Function):
    """The bias row v w^T of the columns whose input v is the same for every point, broadcast to n points; gradients from the column
    sums of the rounded output gradient."""

    @staticmethod
    def forward(ctx, v, w, n):
        ctx.save_for_backward(v, w)
        return F.linear(v.reshape(1, -1), w).expand(n, -1)

    @staticmethod
    def backward(ctx, g):
        v, w = ctx.saved_tensors
        cs = _r16_scaled(g).sum(0)
        return (cs @ w).reshape(v.shape), torch.outer(cs, v.reshape(-1)), None


class _NarrowTC(Function):
    """y = x w^T in full precision; dW sees the fp16 copy of x."""

    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return F.linear(x, w)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        return g @ w, g.t() @ _r16(x)


def _wide(x, fold, w, rounding):
    """One wide layer: x [n, K] the per-point inputs (columns 0..K-1 of w), fold the per-call vector behind them (or None)."""
    if not rounding:
        return F.linear(x if fold is None else torch.cat([x, fold.reshape(1, -1).repeat(x.shape[0], 1)], dim=-1), w)
    k = x.shape[1]
    y = _WideTC.apply(x, w[:, :k])
    return y if fold is None else y + _FoldTC.apply(fold, w[:, k:], x.shape[0])


def _narrow(x, w, rounding):
    return _NarrowTC.apply(x, w) if rounding else F.linear(x, w)


def field_forward(params, hp, xyzs, dirs, cond_feat, individual_code, rounding=True, trace=None):
    """(sigma [N] raw, color [N,3], ambient_pos [N,A]) in the weights' dtype; trace as in the module docstring."""
    bound = hp["bound"]
    pls = float(np.exp2(np.log2(hp["desired_resolution"] * bound / 16) / 15))
    pls_amb = float(np.exp2(np.log2(hp["desired_resolution"] / 16) / 15))
    W = lambda net, i: params[f"{net}.net.{i}.weight"]
    dt = W("sigma_net", 0).dtype
    pre = []

    def relu(x):
        pre.append(x.detach())
        return F.relu(x)

    pos_feat = ft._grid(params, hp, "position_embedder", xyzs.float(), bound, pls).to(dt)
    h = relu(_wide(pos_feat, cond_feat, W("ambient_net", 0), rounding))
    h = relu(_wide(h, None, W("ambient_net", 1), rounding))
    amb = torch.tanh(_narrow(h, W("ambient_net", 2), rounding))
    amb_feat = ft._grid(params, hp, "ambient_embedder", amb, 1, pls_amb).to(dt)
    h = relu(_wide(torch.cat([pos_feat, amb_feat], dim=-1), None, W("sigma_net", 0), rounding))
    h = relu(_wide(h, None, W("sigma_net", 1), rounding))
    if rounding:
        h0, geo = _narrow(h, W("sigma_net", 2)[:1], True)[..., 0], _wide(h, None, W("sigma_net", 2)[1:], True)
    else:
        h = F.linear(h, W("sigma_net", 2))
        h0, geo = h[..., 0], h[..., 1:]
    sigma = ft.trunc_exp(h0)
    dfeat = ops.sh_encode(dirs, 4).to(dt)
    h = relu(_wide(torch.cat([dfeat, geo], dim=-1), individual_code, W("color_net", 0), rounding))
    color = torch.sigmoid(_narrow(h, W("color_net", 1), rounding))
    if trace is not None:
        trace["relu_pre"] = pre
    return sigma, color, amb
