"""Each kernel of the SR head (csrc/sr_kernel.cu) against oracle/sr_emulate.layer_f64 -- the same operation in float64 --
fed with that kernel's OWN input read back from the workspace (the rgb input, x0a, x0b, or x1a with img0), so an error
never carries from one layer to the next, at every input size the C ABI accepts (in_res a multiple of 128, up to 1024).

fp16 outputs (x0a of k_sr_conv_in, x0b of k_sr_conv<0>, x1a of k_sr_conv<1>): with v the float64 value and h the kernel's,
  * every element: |h - v| <= 1/2 ulp16(|v| + E) + E, E = c 2^-23 S, S = sum |x w| + |noise| + |bias|.  c bounds the fp32
    arithmetic between the exact sum and the fp16 store.  The accumulation: k_sr_conv_in adds its 27 terms with RN FFMAs
    (<= 27 x 2^-24 S); the wgmma layers add the exact fp16 products in K/16 steps of 16 to an fp32 accumulator, and the
    tensor cores' alignment and normalisation are not assumed to round to nearest: at most 2 x 2^-23 S per step (one unit
    of the 2^-23 place for the alignment of the step's terms, one for the accumulator's rounding), K/8 x 2^-23 S in all.
    The epilogue rounds four times, (acc + noise), + bias, x 0.2f, x sqrt2 (<= 2 x 2^-23 S), and the activation's slope
    (at most fl32(sqrt 2)) scales everything before it.  So c = sqrt2 (27/2 + 2) for k_sr_conv_in and sqrt2 (K/8 + 2) for
    the wgmma layers (K = 1152, 1152, 576).  The bound catches a wrong element (layout, border, frame, noise);
  * h == RN16(v) on at least a set fraction of the elements, and the mean of sign(v) (h - v) / ulp16(v) stays in a small band
    around 0.  These two catch a directed rounding: round-toward-zero misses RN16 on about half the elements that are not
    representable and moves the mean to about -1/2, where the bound above still holds.
fp32 outputs (img0 of k_sr_conv<0>; the image of k_sr_conv<2>): the activations feeding toRGB are never stored, so the bound
  carries E through toRGB: sum_c |rgb_w_c| E_c, + the fp32 error of the 128- / 64-term dot product and its bias
  ((C + 2) 2^-24 sum |terms|), + the skip (four FMAs of exact weights) and the final sum (6 x 2^-24 (|skip| + sum |terms|)).
  The mean of |error| / bound must stay small: an fp16 rounding anywhere in that path (toRGB fed with the rounded
  activation, weights packed with another rounding) is far below the bound per pixel but moves that mean by an order of
  magnitude.
uint8 frames: equal to (int)(clamp(image) * 255) of the same call's fp32 image, everywhere.  Determinism: repeated calls are
bit-identical (the SR kernels use no atomics), with and without the clamp / the video output.

The bars of the fraction, the band and the mean ratio sit at about twice the distance measured on an H100 (see BARS).
Every case prints the edges it is there for and asserts that it reaches them."""
import ctypes
import time

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.superres import Superresolution
from oracle.sr_emulate import layer_f64, rn16, ulp16

pytestmark = pytest.mark.gpu

K = {"in": 27, 0: 1152, 1: 1152, 2: 576}
C_ACC = {l: np.sqrt(2.0) * ((k / 2 if l == "in" else k / 8) + 2) for l, k in K.items()}
COUT = {0: 128, 2: 64}
# H100 80GB HBM3 (700 W), worst over the cases below: == RN16(v) on 0.99953 / 0.99417 / 0.99506 of the elements of
# x0a / x0b / x1a; sign-weighted mean within +-0.00017 / 0.00207 / 0.00167 ulp16 (the tensor-core layers lean toward zero);
# mean fp32 error / bound 0.00040 (img0), 0.00059 (image).  Each bar sits at about twice that distance.
BARS = {
    "frac": {"in": 0.999, 0: 0.988, 1: 0.99},     # least fraction of fp16 outputs equal to RN16(v)
    "band": {"in": 0.0005, 0: 0.005, 1: 0.003},   # |mean of sign(v) (h - v) / ulp16(v)|
    "ratio": {0: 0.001, 2: 0.0012},               # mean of |fp32 error| / its bound
}


def _state(loud):
    shapes = {k: tuple(v.shape) for k, v in Superresolution(channels=3).state_dict().items()}
    st = scn.synthetic_sr_state(shapes, seed=3)          # the state of tests/golden/sr_head.npz
    if loud:
        # per layer: a quarter of the channels biased past the +256 clamp, a quarter onto the leaky branch, and a quarter with
        # weights 1e-10 x the others (demodulation's 1e-8 then keeps them tiny) and no bias: fp16 subnormals
        for name in ("block0.conv0", "block0.conv1", "block1.conv0", "block1.conv1"):
            b, w = st[name + ".bias"].clone(), st[name + ".weight"].clone()
            b[0::4], b[1::4], b[2::4] = 320.0, -60.0, 0.0
            w[2::4] *= 1e-10
            st[name + ".bias"], st[name + ".weight"] = b, w
    return st


def _net(loud=False):
    net = Superresolution(channels=3).eval()
    net.load_state_dict(_state(loud), strict=False)
    return net.cuda()


def _frames(F, R):
    """Adjacent frames differ by O(1): hashed, its complement, all zero, all one, another hash."""
    a = scn.hashed_uniform(R * R * 3, 78, 1.0).reshape(R, R, 3) + 0.5
    b = scn.hashed_uniform(R * R * 3, 79, 1.0).reshape(R, R, 3) + 0.5
    pool = [a, 1.0 - a, torch.zeros_like(a), torch.ones_like(a), b]
    return torch.stack([pool[i % 5] for i in range(F)]).cuda()


def _noise(kind, F, R, seed):
    """kind: 'none' (a NULL array), 'shared' ([res,res] planes, noise_per_frame 0), 'frame' (N(0, 0.5^2) per frame and layer),
    'mixed' (per-frame planes on layers 0 and 3, NULL on 1 and 2).  Returns (planes, noise_per_frame)."""
    if kind == "none":
        return None, 0
    g = torch.Generator(device="cuda").manual_seed(seed)
    res = [R, R, 2 * R, 2 * R]
    if kind == "shared":
        return [torch.randn(r, r, generator=g, device="cuda") * 0.5 for r in res], 0
    planes = [torch.randn(F, r, r, generator=g, device="cuda") * 0.5 for r in res]
    if kind == "mixed":
        planes[1] = planes[2] = None
    return planes, 1


def _layout(F, R):
    """Mirror of sr_work_layout (capi.cu): x0a, x0b fp16 [F,R,R,128], img0 fp32 [F,R,R,3], x1a fp16 [F,2R,2R,64], 256-byte
    aligned in that order."""
    px, o, out = F * R * R, 0, {}
    for name, nbytes in (("x0a", px * 256), ("x0b", px * 256), ("img0", px * 12), ("x1a", px * 512)):
        out[name] = (o, nbytes)
        o += (nbytes + 255) // 256 * 256
    return out, o


def _views(ws, F, R):
    lay, _ = _layout(F, R)
    shp = {"x0a": ((F, R, R, 128), torch.float16), "x0b": ((F, R, R, 128), torch.float16),
           "img0": ((F, R, R, 3), torch.float32), "x1a": ((F, 2 * R, 2 * R, 64), torch.float16)}
    return {k: ws[o:o + n].view(shp[k][1]).view(shp[k][0]) for k, (o, n) in lay.items()}


def _call(net, rgb, planes, per_frame, R, ws, out, clamp01=0, u8=None):
    st = net._native_state()
    L = _capi.lib()
    arr = None
    if planes is not None:
        arr = (_capi.c_void_p * 4)()
        for i, p in enumerate(planes):
            arr[i] = _capi.ptr(p, torch.float32) if p is not None else None
        arr = ctypes.byref(arr)
    F = rgb.shape[0]
    if u8 is None:
        rc = L.gfpp_sr_forward(ctypes.byref(st["model"]), F, R, _capi.ptr(rgb), arr, per_frame, _capi.ptr(out), clamp01,
                               _capi.ptr(ws), ws.numel(), _capi.stream_ptr())
    else:
        rc = L.gfpp_sr_forward_video(ctypes.byref(st["model"]), F, R, _capi.ptr(rgb), arr, per_frame, _capi.ptr(out),
                                     _capi.ptr(u8), _capi.ptr(ws), ws.numel(), _capi.stream_ptr())
    _capi.check(rc, "sr_forward")


def check_fp16(tag, layer, h, ref):
    """h: the kernel's fp16 output, ref: layer_f64's dict for the same elements."""
    v, h = ref["v"], h.double()
    E = C_ACC[layer] * 2.0 ** -23 * ref["S"]
    d = (h - v).abs()
    u = ulp16(v)
    past = (d - 0.5 * ulp16(v.abs() + E)).clamp(min=0.0)     # the error past the fp16 rounding: within E
    nz = v != 0
    frac = (h == rn16(v)).double().mean().item()
    mean = ((torch.sign(v) * (h - v) / u)[nz]).mean().item()
    worst = torch.where(past > 0, past / E, past).max().item()
    print(f"  {tag} {layer!s:>2}: max |h - v| {(d / u).max().item():.3f} ulp16, past 1/2 ulp16 {worst:.3f} E at most, "
          f"== RN16(v) {frac:.5f}, sign-weighted mean {mean:+.5f} ulp16")
    assert worst <= 1.0, (tag, layer, worst)
    assert frac >= BARS["frac"][layer], (tag, layer, frac)
    assert abs(mean) <= BARS["band"][layer], (tag, layer, mean)
    return v


def check_fp32(tag, layer, got, ref):
    """got: the kernel's fp32 img0 / image (NHWC) for ref's elements."""
    B = (C_ACC[layer] * 2.0 ** -23 * ref["rgbS"] + (COUT[layer] + 2) * 2.0 ** -24 * ref["dot"]
         + 6 * 2.0 ** -24 * (ref["skip"] + ref["dot"]))
    err = (got.double() - ref["img"]).abs()
    r = torch.where(err > 0, err / B, err)
    print(f"  {tag} {layer!s:>2}: fp32 max |err| {err.max().item():.3e} against bound {B.max().item():.3e}; "
          f"max err / bound {r.max().item():.4f}, mean {r.mean().item():.5f}")
    assert r.max().item() <= 1.0, (tag, layer, r.max().item())
    assert r.mean().item() <= BARS["ratio"][layer], (tag, layer, r.mean().item())


def _edges(v, layer, counts):
    a = v.abs()
    counts.setdefault(layer, [0, 0, 0])
    counts[layer][0] += int((a == 256.0).sum())
    counts[layer][1] += int((v < 0).sum())
    counts[layer][2] += int(((a > 0) & (a < 2.0 ** -14)).sum())


CASES = [
    # id, in_res, frames, noise, loud state, rows (None: every row)
    ("r128_f1_null", 128, 1, "none", False, None),
    ("r256_f5_frame", 256, 5, "frame", False, None),
    ("r384_f2_shared", 384, 2, "shared", False, None),
    ("r256_f2_mixed_loud", 256, 2, "mixed", True, None),
    ("r640_f1_shared_loud", 640, 1, "shared", True, None),
    ("r1024_f2_mixed_rows", 1024, 2, "mixed", False, "subset"),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sr_kernels_against_float64_per_layer(case):
    tag, R, F, kind, loud, rows = case
    t0 = time.time()
    L = _capi.lib()
    net = _net(loud)
    fw = net._native_state()["fw"]
    rgb = _frames(F, R)
    planes, per_frame = _noise(kind, F, R, seed=R + F)
    lay, total = _layout(F, R)
    assert total == L.gfpp_sr_workspace_bytes(F, R), "the workspace mirror drifted from sr_work_layout"

    # ---- the edges this case is for
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {0: F * R * R // 128, 1: F * R * R // 128, 2: F * 4 * R * R // 128}
    ctas = {l: min(sms * (1 if l == 1 else 2), tiles[l]) for l in tiles}
    print(f"\n[{tag}] in_res {R}: {R // 128} tile(s) per row; tiles {tiles}, CTAs {ctas}; workspace {total / 2 ** 30:.2f} GiB")
    if R == 128 and F == 1:
        assert tiles[0] < sms * 2 and tiles[1] < sms, "blocks = n_tiles path"
    if R in (384, 640):   # an odd number of tiles per row: consecutive tiles of a CTA land on different rows and x offsets
        assert (R // 128) % 2 == 1 and R // 128 > 1
    if F == 5:
        per_cta = tiles[2] / ctas[2]
        print(f"[{tag}] k_sr_conv<2>: {per_cta:.1f} tiles per CTA, the 4-deep weight ring turns {per_cta * 9 / 4:.0f} times")
        assert per_cta > 30
    if F > 1:
        jump = min((rgb[i] - rgb[i + 1]).abs().mean().item() for i in range(F - 1))
        print(f"[{tag}] least mean |frame i - frame i+1| = {jump:.3f}")
        assert jump > 0.25
    x1a_lo, x1a_hi = lay["x1a"][0], lay["x1a"][0] + lay["x1a"][1]
    if R == 1024:
        print(f"[{tag}] x1a spans bytes [{x1a_lo}, {x1a_hi}) of the workspace: across 2^31 = {2 ** 31}")
        assert x1a_lo < 2 ** 31 < x1a_hi
    if planes is None:
        print(f"[{tag}] noise: NULL array")
    else:
        print(f"[{tag}] noise planes {[None if p is None else tuple(p.shape) for p in planes]}, noise_per_frame {per_frame}")

    # ---- three calls: fp32 image, the same again, then clamped image + uint8 frames
    ws = torch.empty(total, dtype=torch.uint8, device="cuda")
    ws2 = torch.empty_like(ws)
    raw = torch.empty(F, 3, 2 * R, 2 * R, device="cuda")
    raw2, clamped = torch.empty_like(raw), torch.empty_like(raw)
    u8 = torch.empty(F, 2 * R, 2 * R, 3, dtype=torch.uint8, device="cuda")
    _call(net, rgb, planes, per_frame, R, ws, raw)
    _call(net, rgb, planes, per_frame, R, ws2, raw2)
    torch.cuda.synchronize()
    assert torch.equal(ws, ws2) and torch.equal(raw.view(torch.int32), raw2.view(torch.int32)), "two identical calls differ"
    del raw2
    _call(net, rgb, planes, per_frame, R, ws2, clamped, u8=u8)
    torch.cuda.synchronize()
    assert torch.equal(ws, ws2), "the workspace depends on the output mode"
    del ws2
    assert torch.equal(clamped, raw.clamp(0.0, 1.0))
    assert torch.equal(u8, (clamped.permute(0, 2, 3, 1) * 255.0).to(torch.int32).to(torch.uint8)), "uint8 frames"
    del clamped, u8

    # ---- per-layer pins
    w = _views(ws, F, R)
    if rows is None:
        r_in, r_out = torch.arange(R), torch.arange(2 * R)
    else:
        # first and last two rows of every frame, the x1a rows whose bytes straddle 2^31, 8 seeded rows
        row_bytes = 2 * R * 64 * 2
        g = (2 ** 31 - x1a_lo) // row_bytes                   # global x1a row (frame * 2R + Y) holding byte 2^31
        straddle = sorted({g - 1, g} if (2 ** 31 - x1a_lo) % row_bytes == 0 else {g})
        assert all(0 <= s < F * 2 * R for s in straddle)
        Ys = [s % (2 * R) for s in straddle]
        print(f"[{tag}] x1a rows at byte 2^31 (frame, row): {[(s // (2 * R), s % (2 * R)) for s in straddle]}")
        seeded = torch.randint(0, R, (8,), generator=torch.Generator().manual_seed(11)).tolist()
        r_in = torch.tensor(sorted({0, 1, R - 2, R - 1, *[Y // 2 for Y in Ys], *seeded}))
        r_out = torch.tensor(sorted({0, 1, 2 * R - 2, 2 * R - 1, *Ys, *[2 * s for s in seeded]}))
    n_in = planes[0] if planes is not None else None
    counts = {}
    rgb_out = raw.permute(0, 2, 3, 1)
    ref = layer_f64(fw, "in", rgb, n_in, rows=r_in)
    _edges(check_fp16(tag, "in", w["x0a"][:, r_in.cuda()], ref), "in", counts)
    ref = layer_f64(fw, 0, w["x0a"], planes[1] if planes else None, skip=rgb, rows=r_in)
    _edges(check_fp16(tag, 0, w["x0b"][:, r_in.cuda()], ref), 0, counts)
    check_fp32(tag, 0, w["img0"][:, r_in.cuda()], ref)
    ref = layer_f64(fw, 1, w["x0b"], planes[2] if planes else None, rows=r_in)
    r_up = torch.stack([2 * r_in, 2 * r_in + 1], 1).reshape(-1)
    _edges(check_fp16(tag, 1, w["x1a"][:, r_up.cuda()], ref), 1, counts)
    ref = layer_f64(fw, 2, w["x1a"], planes[3] if planes else None, skip=w["img0"], rows=r_out)
    _edges(ref["v"], 2, counts)
    check_fp32(tag, 2, rgb_out[:, r_out.cuda()], ref)
    del ref
    print(f"[{tag}] per layer (clamped at 256, negative, fp16 subnormal): {counts}")
    if loud:
        for layer, c in counts.items():
            assert min(c) > 0, (layer, c)
    del ws, w, raw, rgb_out
    torch.cuda.empty_cache()
    print(f"[{tag}] {time.time() - t0:.1f} s")
