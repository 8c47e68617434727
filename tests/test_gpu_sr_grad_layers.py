"""Each backward kernel of the SR head (csrc/sr_train_kernel.cu) against float64 on its OWN inputs: the activations of the
training forward and the gradients of the previous backward stage are read back from the saved buffer and the backward's
workspace, so an error never carries from one kernel to the next.  in_res 128 / 256 / 512, up to 3 frames, noise NULL / shared /
per-frame, the plain state and a loud one (clamp and leaky branch live).

Model of the kernels' arithmetic (v: the float64 value on the kernel's inputs, h: the kernel's):
  * The tensor-core products (dgrad of the three GEMM layers, their weight gradients) take the gradient operand rounded to
    nearest-even tf32 (modelled exactly: `tf32` below) and the fp16 weights / activations of the forward (exact).  So v is the
    exact sum of exact products.  The fp32 accumulation adds K / 8 k-steps of 8; the tensor cores' alignment and normalisation
    are not assumed to round to nearest, so each step may cost 2 x 2^-23 S (S = sum |terms|), K / 4 x 2^-23 S in all.  The
    epilogue rounds at most four more times (toRGB0's three FMAs, the slope), and the slope (at most fl32(sqrt 2)) scales it.
    Bound: |h - v| <= sqrt2 (K / 4 + 4) 2^-23 S.  For the weight gradients K is the pixels of a slice and the fixed-order sum
    of the slices adds (slices + 2) 2^-24 S.
  * The CUDA-core stages (toRGB adjoints, the skip's adjoint, the input layer's dgrad and wgrad, the bias / noise / toRGB sums)
    round to nearest in fp32: (n + 2) 2^-24 S for n terms in sequence.
  * The toRGB stages rebuild the toRGB output r from the fp16-stored activation (the forward used the fp32 value before its
    fp16 store), so the model takes the stored one too; pixels whose |r| is within the fp32 error of r of the clamp at 256 are
    left out of the element check (either side of the mask is right there).
A wrong tap, phase, border, frame or layout breaks the element bound.  A directed rounding of the gradient operand (truncation
to tf32 instead of RN) stays near that bound per element but moves the mean of |h - v| / bound by far more than MEAN_RATIO,
which sits at about twice the worst measured on an H100 SXM (80 GB, 700 W).  Repeated calls are bit-identical."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from genefaceplusplus_b200 import _capi, scene as scn
from genefaceplusplus_b200.superres import Superresolution, _binomial_filter, _upsample2x

pytestmark = pytest.mark.gpu

U23, U24 = 2.0 ** -23, 2.0 ** -24
S1 = float(np.float32(np.sqrt(2.0)))
S2 = float(np.float32(np.float32(0.2) * np.float32(np.sqrt(2.0))))
MEAN_RATIO = 0.05
SLICES = {"conv1_w": 64, "up_w": 16, "conv0_w": 32}


def tf32(x):
    """fp32 -> nearest-even tf32 (10 mantissa bits), as fp32."""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0xFFF + ((b >> 13) & 1)) & 0xFFFFE000
    return torch.where(b >= 2 ** 31, b - 2 ** 32, b).to(torch.int32).view(torch.float32)


def dact(y):
    return torch.where(y.abs() < 256, torch.where(y > 0, torch.full_like(y, S1), torch.full_like(y, S2)), torch.zeros_like(y))


def _net(loud):
    net = Superresolution(channels=3)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    st = scn.synthetic_sr_state(shapes, seed=3)
    if loud:
        for name in ("block0.conv0", "block0.conv1", "block1.conv0", "block1.conv1"):
            b, w = st[name + ".bias"].clone(), st[name + ".weight"].clone()
            b[0::4], b[1::4], b[2::4] = 320.0, -60.0, 0.0
            w[2::4] *= 1e-10
            st[name + ".bias"], st[name + ".weight"] = b, w
    net.load_state_dict(st, strict=False)
    return net.cuda()


def _views(buf, F, R, names):
    """Slices of a byte buffer laid out as consecutive 256-byte-rounded blocks (capi.cu's Bump)."""
    px = F * R * R
    sizes = {"x0a": px * 256, "x0b": px * 256, "img0": px * 12, "x1a": px * 512, "x1b": px * 512,
             "wt0": 147456, "wt1": 1179648, "wt2": 589824, "g1": px * 1024, "gup": px * 1024, "g0": px * 512, "gin": px * 512,
             "gimg0": px * 12, "gr0": px * 12}
    out, off = {}, 0
    for n in names:
        out[n] = buf[off:off + sizes[n]]
        off += (sizes[n] + 255) // 256 * 256
    return out


def _check(tag, name, h, v, bound, keep=None, stats=None, directed=False):
    h, v, bound = h.double(), v.double(), bound.double()
    err = (h - v).abs()
    if keep is not None:
        err, bound = err[keep], bound[keep]
    bound = bound + 1e-300
    worst = float((err / bound).max())
    mean = float((err / bound).mean())
    stats[name] = (worst, mean)
    assert worst <= 1.0, (tag, name, worst)
    if directed:   # the tensor-core products: where a truncated tf32 operand would show
        assert mean <= MEAN_RATIO, (tag, name, mean)


CASES = [("r128_f1_null_loud", 128, 1, "none", True), ("r256_f3_frame", 256, 3, "frame", False),
         ("r512_f1_shared_loud", 512, 1, "shared", True), ("r256_f2_shared_loud", 256, 2, "shared", True)]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_backward_kernels_against_float64(case):
    tag, R, F, kind, loud = case
    L = _capi.lib()
    net = _net(loud)
    st = net._native_state()
    fw = st["fw"]
    g = torch.Generator(device="cuda").manual_seed(R + F)
    rgb = (torch.rand(F, R * R, 3, generator=g, device="cuda"))
    res = [R, R, 2 * R, 2 * R]
    if kind == "none":
        planes = raws = None
    elif kind == "shared":
        raws = [torch.randn(r, r, generator=g, device="cuda") for r in res]
    else:
        raws = [torch.randn(F, r, r, generator=g, device="cuda") for r in res]
    per_frame = 1 if kind == "frame" else 0
    if raws is not None:
        planes = [r * 0.3 for r in raws]
        arr, rarr = (ctypes.c_void_p * 4)(*[p.data_ptr() for p in planes]), (ctypes.c_void_p * 4)(*[r.data_ptr() for r in raws])
    G = torch.randn(F, 3, 2 * R, 2 * R, generator=g, device="cuda") / (F * 3 * 4 * R * R)

    out = torch.empty(F, 3, 2 * R, 2 * R, device="cuda")
    saved = torch.empty(L.gfpp_sr_train_workspace_bytes(F, R), dtype=torch.uint8, device="cuda")
    _capi.check(L.gfpp_sr_forward_train(ctypes.byref(st["model"]), F, R, rgb.data_ptr(), None if raws is None else ctypes.byref(arr),
                                        per_frame, out.data_ptr(), saved.data_ptr(), saved.numel(), None), "gfpp_sr_forward_train")
    sizes = [27 * 128, 128 * 1152, 256 * 1152, 64 * 576, 128, 128, 64, 64, 4, 384, 192, 3, 3]
    runs = []
    for _ in range(2):
        flat = torch.empty(sum(sizes), device="cuda")
        parts = list(torch.split(flat, sizes))
        gd = _capi.SrGrad()
        gd.conv_in_w, gd.conv0_w, gd.up_w, gd.conv1_w = (t.data_ptr() for t in parts[:4])
        for i in range(4):
            gd.bias[i] = parts[4 + i].data_ptr()
        gd.noise_strength = parts[8].data_ptr()
        for i in range(2):
            gd.rgb_w[i], gd.rgb_b[i] = parts[9 + i].data_ptr(), parts[11 + i].data_ptr()
        grad_in = torch.empty_like(rgb)
        ws = torch.empty(L.gfpp_sr_backward_workspace_bytes(F, R), dtype=torch.uint8, device="cuda")
        _capi.check(L.gfpp_sr_backward(ctypes.byref(st["model"]), F, R, rgb.data_ptr(), saved.data_ptr(), saved.numel(),
                                       None if raws is None else ctypes.byref(rarr), per_frame, G.data_ptr(), grad_in.data_ptr(),
                                       ctypes.byref(gd), ws.data_ptr(), ws.numel(), None), "gfpp_sr_backward")
        torch.cuda.synchronize()
        runs.append((flat, grad_in, ws))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), "two identical backward calls differ"
    flat, grad_in, ws = runs[0]
    parts = dict(zip(["conv_in_w", "conv0_w", "up_w", "conv1_w", "b0", "b1", "b2", "b3", "ns", "rgbw0", "rgbw1", "rgbb0", "rgbb1"],
                     torch.split(flat, sizes)))

    sv = _views(saved, F, R, ["x0a", "x0b", "img0", "x1a", "x1b"])
    wk = _views(ws, F, R, ["wt0", "wt1", "wt2", "g1", "gup", "g0", "gin", "gimg0", "gr0"])
    h16 = lambda t, C, r: t.view(torch.float16).view(F, r, r, C).double()       # noqa: E731
    f32 = lambda t, C, r: t.view(torch.float32).view(F, r, r, C)                # noqa: E731
    x0a, x0b, x1a, x1b = h16(sv["x0a"], 128, R), h16(sv["x0b"], 128, R), h16(sv["x1a"], 64, 2 * R), h16(sv["x1b"], 64, 2 * R)
    g1, gup, g0, gin = f32(wk["g1"], 64, 2 * R), f32(wk["gup"], 64, 2 * R), f32(wk["g0"], 128, R), f32(wk["gin"], 128, R)
    gimg0, gr0 = f32(wk["gimg0"], 3, R), f32(wk["gr0"], 3, R)
    d = lambda t: t.double().cuda()                                              # noqa: E731
    rw0, rw1, rb0, rb1 = d(fw["rgb_w"][0]), d(fw["rgb_w"][1]), d(fw["rgb_b"][0]), d(fw["rgb_b"][1])
    W16 = lambda m, co, ci: d(m).half().double().view(co, 3, 3, ci).permute(0, 3, 1, 2)   # noqa: E731
    stats = {}

    # ---- k_srb_rgb<64>: toRGB1 adjoint times y'(x1b) at 2R
    Gn = G.double().permute(0, 2, 3, 1)                                          # [F,2R,2R,3]
    r1 = x1b @ rw1.T + rb1
    r1_err = 66 * U24 * (x1b.abs() @ rw1.abs().T + rb1.abs())
    m1 = (r1.abs() < 256).double()
    gr1 = Gn * m1
    v = (gr1 @ rw1) * dact(x1b)
    keep1 = ((r1.abs() - 256).abs() > r1_err).all(-1)
    S = (gr1.abs() @ rw1.abs()) * S1
    _check(tag, "g1", g1, v, 5 * U24 * S + 1e-45, keep1[..., None].expand_as(v), stats)

    # ---- k_srb_rgb<128>: adjoint of the up-sampled skip, toRGB0's clamp mask
    f = _binomial_filter().double().cuda()
    z = torch.zeros(F, 3, R, R, dtype=torch.float64, device="cuda", requires_grad=True)
    (vimg,) = torch.autograd.grad(_upsample2x(z, f), z, G.double())
    (simg,) = torch.autograd.grad(_upsample2x(z, f), z, G.double().abs())
    vimg, simg = vimg.permute(0, 2, 3, 1), simg.permute(0, 2, 3, 1)
    _check(tag, "g_img0", gimg0, vimg, 18 * U24 * simg + 1e-45, None, stats)
    r0 = x0b @ rw0.T + rb0
    r0_err = 130 * U24 * (x0b.abs() @ rw0.abs().T + rb0.abs())
    keep0 = ((r0.abs() - 256).abs() > r0_err)
    assert torch.equal(gr0[keep0], (gimg0 * (r0.abs() < 256))[keep0].float()), "g_r0 is g_img0 masked by toRGB0's clamp"

    # ---- dgrad of block1.conv1 (K = 576), block1.conv0 (K = 2304), block0.conv1 (K = 1152)
    def dgrad(A, W, act, K, extra=None, extra_abs=None):
        a = tf32(A.contiguous()).double().permute(0, 3, 1, 2)
        v = Fn.conv_transpose2d(a, W, padding=1).permute(0, 2, 3, 1)
        s = Fn.conv_transpose2d(a.abs(), W.abs(), padding=1).permute(0, 2, 3, 1)
        if extra is not None:
            v, s = v + extra, s + extra_abs
        sl = dact(act)
        return v * sl, np.sqrt(2.0) * (K / 4 + 4) * U23 * s * sl.clamp_min(S2) + 1e-45

    v, b = dgrad(g1, W16(fw["conv1_w"], 64, 64), x1a, 576)
    _check(tag, "dgrad conv1", gup, v, b, None, stats, True)
    ph = lambda t: t.view(F, R, 2, R, 2, 64).permute(0, 1, 3, 2, 4, 5).reshape(F, R, R, 256)   # noqa: E731
    gr0d = gr0.double()
    v, b = dgrad(ph(gup), W16(fw["up_w"], 256, 128), x0b, 2304, gr0d @ rw0, gr0d.abs() @ rw0.abs())
    _check(tag, "dgrad up", g0, v, b, None, stats, True)
    v, b = dgrad(g0, W16(fw["conv0_w"], 128, 128), x0a, 1152)
    _check(tag, "dgrad conv0", gin, v, b, None, stats, True)

    # ---- block0.conv0 (128 -> 3) dgrad on CUDA cores, + g_img0
    Win = d(fw["conv_in_w"]).view(3, 3, 3, 128).permute(3, 2, 0, 1)
    a = gin.double().permute(0, 3, 1, 2)
    v = Fn.conv_transpose2d(a, Win, padding=1).permute(0, 2, 3, 1) + gimg0.double()
    s = Fn.conv_transpose2d(a.abs(), Win.abs(), padding=1).permute(0, 2, 3, 1) + gimg0.double().abs()
    _check(tag, "dgrad in", grad_in.view(F, R, R, 3), v, 1154 * U24 * s + 1e-45, None, stats)

    # ---- weight gradients
    def wgrad(x, A, co, ci, key, round_a=True):
        xx = x.permute(0, 3, 1, 2)
        a = (tf32(A.contiguous()) if round_a else A).double().permute(0, 3, 1, 2)
        v = torch.nn.grad.conv2d_weight(xx, (co, ci, 3, 3), a, padding=1)
        s = torch.nn.grad.conv2d_weight(xx.abs(), (co, ci, 3, 3), a.abs(), padding=1)
        K = F * x.shape[1] * x.shape[2] // SLICES.get(key, 256) if round_a else None
        bnd = ((K / 4 + 4) * U23 + (SLICES[key] + 2) * U24) if round_a else None
        return v, s, bnd

    for key, x, A, co, ci in (("conv1_w", x1a, g1, 64, 64), ("up_w", x0b, ph(gup), 256, 128), ("conv0_w", x0a, g0, 128, 128)):
        v, s, c = wgrad(x, A, co, ci, key)
        v, s = v.permute(0, 2, 3, 1).reshape(co, 9 * ci), s.permute(0, 2, 3, 1).reshape(co, 9 * ci)
        _check(tag, "wgrad " + key, parts[key].view(co, 9 * ci), v, c * s + 1e-45, None, stats, True)
    v, s, _ = wgrad(rgb.view(F, R, R, 3).double(), gin, 128, 3, "conv_in_w", round_a=False)
    n = F * R * R // 256 + 256 + 2
    _check(tag, "wgrad conv_in_w", parts["conv_in_w"].view(27, 128), v.permute(2, 3, 1, 0).reshape(27, 128),
           n * U24 * s.permute(2, 3, 1, 0).reshape(27, 128) + 1e-45, None, stats)

    # ---- biases and noise strengths (sum over pixels of the pre-activation gradient, and of it times the raw plane)
    for i, (gp, r) in enumerate(((gin, R), (g0, R), (gup, 2 * R), (g1, 2 * R))):
        gd64 = gp.double().reshape(F, r * r, -1)
        n = F * r * r // 256 + 256 + 2
        _check(tag, f"bias{i}", parts[f"b{i}"], gd64.sum((0, 1)), n * U24 * gd64.abs().sum((0, 1)) + 1e-45, None, stats)
        if raws is None:
            assert float(parts["ns"][i]) == 0.0
        else:
            rw = raws[i].double().reshape(-1, r * r)
            rw = rw if rw.shape[0] == F else rw.expand(F, -1)
            t = gd64 * rw[..., None]
            _check(tag, f"noise{i}", parts["ns"][i:i + 1], t.sum().view(1), (n + gd64.shape[-1]) * U24 * t.abs().sum().view(1) + 1e-45,
                   None, stats)

    # ---- toRGB weights and biases
    for key, kb, gr, x, C in (("rgbw1", "rgbb1", gr1, x1b, 64), ("rgbw0", "rgbb0", gr0d, x0b, 128)):
        grf, xf = gr.reshape(-1, 3), x.reshape(-1, C)
        n = grf.shape[0] // 256 + 256 + 2
        _check(tag, key, parts[key].view(3, C), grf.T @ xf, n * U24 * (grf.abs().T @ xf.abs()) + 1e-45, None, stats)
        _check(tag, kb, parts[kb], grf.sum(0), n * U24 * grf.abs().sum(0) + 1e-45, None, stats)

    print(f"\n[{tag}] worst / mean |h - v| / bound: " + ", ".join(f"{k} {w:.3f}/{m:.4f}" for k, (w, m) in stats.items()))
    if loud:
        assert float((x1a.abs() >= 256).double().mean()) > 0 and float((x1a < 0).double().mean()) > 0
