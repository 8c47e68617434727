"""oracle/sr_emulate.py -- TEST INFRASTRUCTURE: CPU emulation of the data flow of the native SR-head kernels.

Restates, in plain torch on the CPU, exactly what genefaceplusplus_b200/csrc/sr_kernel.cu computes from the folded GEMM
matrices of `Superresolution.folded_weights()` (the gfpp_sr_desc layouts, include/gfpp.h): NHWC activations rounded to fp16
between the layers, K ordered (tap, channel) with tap = ky*3+kx <-> pixel offset (ky-1, kx-1) and zeros outside the image,
the four output phases of the merged up-sampling layer scattered to (2y+py, 2x+px), fp32 toRGB on the unrounded
activations, the closed-form [1,3,3,1] up-sampling of the rgb skip.  Two uses:

  * on the CPU (tests/test_host_logic.py): against `Superresolution.forward` (the fp32 convolutions pinned by the reference
    golden tests/golden/sr_head.npz) -- proves the folding algebra and every layout convention of the host half;
  * on the GPU (tests/test_gpu_sr_native.py): the kernels must agree with this rounding model to ~1e-5, which separates a
    layout / descriptor / pipeline bug from the expected fp16 operand rounding (~5e-4 against the fp32 path).

`layer_f64` restates ONE kernel in float64 on that kernel's own input (tests/test_gpu_sr_layers.py feeds it the kernels'
workspace, so no rounding carries from one layer to the next; tests/test_oracle_sr_layers.py pins its rounding-free chain to
the module in float64).

Never imported by the package.
"""
import math

import torch
import torch.nn.functional as F


def _r16(x, on):
    return x.half().float() if on else x


def _act(x, noise, bias):
    if noise is not None:
        x = x + noise.reshape(noise.shape[0] if noise.dim() == 3 else 1, noise.shape[-2], noise.shape[-1], 1)
    x = F.leaky_relu(x + bias.view(1, 1, 1, -1), 0.2) * math.sqrt(2.0)
    return x.clamp(-256.0, 256.0)


def _im2col(x):
    """x [F,H,W,C] -> [F,H,W,9*C] with k = (ky*3+kx)*C + c and zeros outside the image."""
    Fn, H, W, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[:, ky:ky + H, kx:kx + W, :] for ky in range(3) for kx in range(3)], dim=-1)


def _phases(u):
    """[F,h,w,256] GEMM output of the up-sampling layer, column (py*2+px)*64 + co -> [F,2h,2w,64] at pixel (2y+py, 2x+px)."""
    Fn, h, w = u.shape[:3]
    return u.reshape(Fn, h, w, 2, 2, 64).permute(0, 1, 3, 2, 4, 5).reshape(Fn, 2 * h, 2 * w, 64)


def _upsample_skip(img):
    """img [F,h,w,3] -> [F,2h,2w,3]: even outputs 0.25*in[i-1] + 0.75*in[i], odd 0.75*in[i] + 0.25*in[i+1] per axis."""
    def up(t, dim):
        n = t.shape[dim]
        z = torch.zeros_like(t.narrow(dim, 0, 1))
        prev = torch.cat([z, t.narrow(dim, 0, n - 1)], dim)
        nxt = torch.cat([t.narrow(dim, 1, n - 1), z], dim)
        even = 0.25 * prev + 0.75 * t
        odd = 0.75 * t + 0.25 * nxt
        return torch.stack([even, odd], dim + 1).flatten(dim, dim + 1)
    return up(up(img, 1), 2)


@torch.no_grad()
def emulate(fw, rgb_flat, R, noise=(None, None, None, None), fp16=True, clamp=False, intermediates=None):
    """fw: folded_weights() dict (CPU tensors); rgb_flat [F, R*R, 3]; noise[i]: None or [res,res] / [F,res,res] planes already
    multiplied by the layer's strength.  Returns [F,3,2R,2R].  `intermediates`: optional dict that receives the tensors the
    kernels keep in their workspace (x0a, x0b: [F,R,R,128]; img0 [F,R,R,3]; x1a [F,2R,2R,64]) for layer-by-layer diagnosis."""
    x = rgb_flat.reshape(-1, R, R, 3).float()
    h = _im2col(x) @ fw["conv_in_w"]                                        # fp32 FFMA layer, [F,R,R,128]
    h = _r16(_act(h, noise[0], fw["bias"][0]), fp16)                        # stored as fp16 NHWC
    x0a = h
    a = _act(_im2col(h) @ _r16(fw["conv0_w"], fp16).t(), noise[1], fw["bias"][1])
    img0 = x + (a @ fw["rgb_w"][0].t() + fw["rgb_b"][0]).clamp(-256.0, 256.0)   # toRGB on the unrounded activations
    h = _r16(a, fp16)
    u = _phases(_im2col(h) @ _r16(fw["up_w"], fp16).t())                    # [F,2R,2R,64]
    x0b = h
    h = _r16(_act(u, noise[2], fw["bias"][2]), fp16)
    if intermediates is not None:
        intermediates.update(x0a=x0a, x0b=x0b, img0=img0, x1a=h)
    a = _act(_im2col(h) @ _r16(fw["conv1_w"], fp16).t(), noise[3], fw["bias"][3])
    img = _upsample_skip(img0) + (a @ fw["rgb_w"][1].t() + fw["rgb_b"][1]).clamp(-256.0, 256.0)
    if clamp:
        img = img.clamp(0.0, 1.0)
    return img.permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------------------------------------ float64, one kernel at a time
F32_SLOPE = float(torch.tensor(0.2, dtype=torch.float32))             # the kernels' 0.2f
F32_SQRT2 = float(torch.tensor(math.sqrt(2.0), dtype=torch.float32))  # and kSqrt2 = fl32(sqrt 2)


def ulp16(v):
    """Spacing of binary16 at float64 v: 2^(e-10) for |v| in [2^e, 2^(e+1)), 2^-24 in the subnormal range (|v| < 2^-14)."""
    _, e = torch.frexp(v)                                                # |v| = m 2^e, m in [0.5, 1)
    e = torch.where(v == 0, torch.full_like(e, -13), e)
    return torch.ldexp(torch.ones_like(v), (e - 1).clamp(min=-14) - 10)


def rn16(v):
    """binary16 round-to-nearest-even of float64 v in ONE rounding (|v| < 65520): v / ulp is exact, torch.round ties to even."""
    u = ulp16(v)
    return torch.round(v / u) * u


def _rows(x, ys):
    """Rows ys of x [F,H,W,C] as float64 [F,n,W,C], zeros for rows outside the image."""
    ok = (ys >= 0) & (ys < x.shape[1])
    t = x[:, ys.clamp(0, x.shape[1] - 1).to(x.device)].double()
    t[:, ~ok.to(x.device)] = 0.0
    return t


@torch.no_grad()
def layer_f64(fw, layer, x, noise=None, skip=None, rows=None, kernel=True, clamp=False, chunk_bytes=1 << 29):
    """What ONE kernel of the SR head computes from its input `x`, in float64, on x's device.

    layer: "in" (k_sr_conv_in: x = the rgb input [F,R,R,3]), 0 (k_sr_conv<0>: x = x0a), 1 (k_sr_conv<1>: x = x0b) or 2
    (k_sr_conv<2>: x = x1a [F,2R,2R,64]); fw: folded_weights(); noise: None or the layer's [res,res] / [F,res,res] plane
    (already times the strength); skip: the rgb input (layer 0) or img0 [F,R,R,3] (layer 2); rows: input-grid rows to compute
    (default all; layer 1 returns output rows 2y and 2y+1 of each).
    kernel=True: the kernels' arithmetic without their roundings -- wgmma weights RN16(fw) (fp32 ones for "in"), exact sums,
    (sum + noise) + bias, leaky-ReLU with 0.2f, times fl32(sqrt 2), clamp to +-256; kernel=False: the module's math (0.2,
    sqrt 2, unrounded weights).  Returns NHWC float64 tensors:
      v       the activation before it is stored as fp16 (x0a, x0b, x1a; for layers 0 and 2 the fp32 input of toRGB)
      S       sum |x w| + |noise| + |bias| per element of v (the scale of its accumulation error)
      img     layers 0 / 2: img0 = skip + clamp(toRGB(v)) / the image = up2(img0) + clamp(toRGB(v)) [, clamped to [0,1]]
      rgbS    sum_c |rgb_w[o,c]| S_c;  dot: sum_c |rgb_w[o,c] v_c| + |rgb_b[o]|;  skip: |the skip term| (bounds of img)
    """
    conv, bi = {"in": ("conv_in_w", 0), 0: ("conv0_w", 1), 1: ("up_w", 2), 2: ("conv1_w", 3)}[layer]
    dev, f64 = x.device, torch.float64
    w = fw[conv].t() if layer == "in" else (fw[conv].half() if kernel else fw[conv])
    w = w.to(dev, f64)
    wa, b = w.abs(), fw["bias"][bi].to(dev, f64)
    slope, gain = (F32_SLOPE, F32_SQRT2) if kernel else (0.2, math.sqrt(2.0))
    Fn, H, W, C = x.shape
    rows = torch.arange(H) if rows is None else torch.as_tensor(rows).reshape(-1)
    if noise is not None:
        noise = noise.to(dev, f64)
    if layer in (0, 2):
        j = 0 if layer == 0 else 1
        rw, rb = fw["rgb_w"][j].to(dev, f64), fw["rgb_b"][j].to(dev, f64)
        sk = skip.to(dev, f64)
        if layer == 2:
            sk, ska = _upsample_skip(sk), _upsample_skip(sk.abs())
        else:
            ska = sk.abs()
    out = {}
    per = max(1, chunk_bytes // (Fn * 3 * W * 9 * C * 8))
    for r in rows.split(per):
        xr = torch.stack([_rows(x, r + dy) for dy in (-1, 0, 1)], 2)                  # [F,n,3,W,C]: rows y-1, y, y+1
        cols = _im2col(xr.reshape(-1, 3, W, C))[:, 1].reshape(Fn, len(r), W, 9 * C)
        s, S = cols @ w.t(), cols.abs() @ wa.t()
        yo = r
        if layer == 1:
            s, S = _phases(s), _phases(S)
            yo = torch.stack([2 * r, 2 * r + 1], 1).reshape(-1)
        if noise is not None:
            nz = noise[..., yo.to(dev), :]
            nz = nz.reshape(nz.shape[0] if nz.dim() == 3 else 1, len(yo), -1, 1)
            s, S = s + nz, S + nz.abs()
        t = s + b
        v = (torch.where(t < 0, slope * t, t) * gain).clamp(-256.0, 256.0)
        part = {"v": v, "S": S + b.abs()}
        if layer in (0, 2):
            rgb = (v @ rw.t() + rb).clamp(-256.0, 256.0)
            img = sk[:, r.to(dev)] + rgb
            part.update(img=img.clamp(0.0, 1.0) if clamp else img, rgbS=part["S"] @ rw.abs().t(),
                        dot=v.abs() @ rw.abs().t() + rb.abs(), skip=ska[:, r.to(dev)])
        for k, t in part.items():
            out.setdefault(k, []).append(t)
    return {k: torch.cat(t, 1) for k, t in out.items()}
