"""Super-resolution head of the SR checkpoints (SURVEY.md 8(f) rank 3): 256x256 NeRF image -> 512x512.

Drop-in for `Superresolution` of modules/radnerfs/radnerf_sr.py:15-48, which the reference assembles from StyleGAN2
synthesis blocks (modules/eg3ds/models/superresolution.py:159-257 `SynthesisBlockNoUp`,
modules/eg3ds/models/networks_stylegan2.py:286-475 `SynthesisLayer` / `ToRGBLayer` / `SynthesisBlock`).  Same parameter and
buffer names and shapes, so `load_state_dict(strict=True)` takes an SR checkpoint as is.  Written from the math, not from
the reference's code:

  * every layer is a style-modulated convolution  y = conv(x, W * s_in * d_out)  with  s = A w + b  (A scaled by
    1/sqrt(w_dim)) and, for the 3x3 layers, the demodulation  d_o = rsqrt(sum_{i,k} (W_oik s_i)^2 + 1e-8);
  * the network always feeds the constant latent w = 1 (radnerf_sr.py:33-34), so s and d are constants of the checkpoint:
    the modulated kernels are built once per call and shared by the whole batch (one plain conv2d per layer for a clip,
    instead of the reference's per-sample grouped convolutions);
  * 3x3 layers: + noise * noise_strength, + bias, leaky-ReLU(0.2) * sqrt(2), clamp to +-256;  1x1 toRGB layers: weights
    scaled by 1/sqrt(C_in), + bias, clamp; the rgb skip path is the input image (block 0) / its 2x FIR up-sampling (block 1);
  * 2x up-sampling convolution (block1.conv0): transposed convolution with stride 2, then the separable binomial filter
    [1,3,3,1]^2 / 64 with gain 4 on the (2H+1)-sized result padded by one pixel -- the polyphase identity the reference's
    conv2d_resample uses (torch_utils/ops/conv2d_resample.py:118-133).

Two implementations live behind `Superresolution.forward`:

  * CUDA tensors, `backend == "native"` (the default): libgfpp's hand-written sm_90a kernels (csrc/sr_kernel.cu through
    gfpp_sr_pack / gfpp_sr_forward): one fp32 FFMA kernel for the 3-channel input layer and three implicit-GEMM wgmma
    kernels with fused noise / bias / leaky-ReLU / clamp / toRGB / skip epilogues; fp16 operands with fp32 accumulation
    (the reference switches these blocks to fp16 on CUDA), toRGB and the skip path fp32.  `folded_weights()` is the host
    half of that path: it folds modulation, demodulation and -- for the up-sampling layer -- the transposed stride-2
    convolution together with its FIR filter into plain GEMM matrices.  A missing libgfpp raises (no silent eager path).
    Under grad, when the input or a parameter requires it, the same kernels run through train_ops.sr_head, whose backward is
    csrc/sr_train_kernel.cu (gfpp_sr_forward_train / gfpp_sr_backward).
  * `backend == "torch"` or CPU tensors: the plain fp32 convolutions below -- the math the goldens pin
    (tests/golden/sr_head.npz) and the checker of the native path (tests/test_gpu_sr_native.py).
"""
import ctypes
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


def _binomial_filter() -> torch.Tensor:
    """[1,3,3,1] (x) [1,3,3,1], normalised to unit DC gain (upfirdn2d.setup_filter([1,3,3,1]))."""
    f = torch.tensor([1.0, 3.0, 3.0, 1.0])
    f = torch.outer(f, f)
    return f / f.sum()


def _fir(x: torch.Tensor, f: torch.Tensor, pad, gain: float) -> torch.Tensor:
    """Depth-wise FIR: pad = (left, right, top, bottom); true convolution with f * gain."""
    c = x.shape[1]
    x = F.pad(x, pad)
    k = (f * gain).flip([0, 1]).to(x.dtype)[None, None].repeat(c, 1, 1, 1)
    return F.conv2d(x, k, groups=c)


def _upsample2x(x: torch.Tensor, f: torch.Tensor) -> torch.Tensor:
    """Zero-insertion by 2 followed by the low-pass f with gain 4 (upfirdn2d.upsample2d): [N,C,H,W] -> [N,C,2H,2W]."""
    n, c, h, w = x.shape
    z = torch.zeros(n, c, h, 2, w, 2, dtype=x.dtype, device=x.device)
    z[:, :, :, 0, :, 0] = x
    return _fir(z.reshape(n, c, 2 * h, 2 * w), f, (2, 1, 2, 1), 4.0)


class _Affine(nn.Module):
    """Style affine: FullyConnectedLayer(w_dim, C, bias_init=1) of networks_stylegan2.py:99-131 with linear activation."""

    def __init__(self, w_dim, channels):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(channels, w_dim))
        self.bias = nn.Parameter(torch.ones(channels))
        self.weight_gain = 1.0 / math.sqrt(w_dim)

    def forward(self, w):  # [w_dim] -> [C]
        return torch.addmv(self.bias, self.weight * self.weight_gain, w)


class _ModConv(nn.Module):
    """3x3 modulated + demodulated convolution layer (SynthesisLayer), optionally 2x up-sampling."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, up=1, conv_clamp=256.0):
        super().__init__()
        self.up, self.resolution, self.conv_clamp = up, resolution, conv_clamp
        self.affine = _Affine(w_dim, in_channels)
        self.weight = nn.Parameter(torch.randn(out_channels, in_channels, 3, 3))
        self.register_buffer("resample_filter", _binomial_filter())
        self.register_buffer("noise_const", torch.randn(resolution, resolution))
        self.noise_strength = nn.Parameter(torch.zeros([]))
        self.bias = nn.Parameter(torch.zeros(out_channels))

    def modulated_weight(self, w):
        s = self.affine(w)                                                   # [I]
        k = self.weight * s.view(1, -1, 1, 1)
        d = (k.square().sum(dim=[1, 2, 3]) + 1e-8).rsqrt()                   # [O]
        return k * d.view(-1, 1, 1, 1)

    def forward(self, x, w, noise_mode="random"):
        k = self.modulated_weight(w).to(x.dtype)
        if self.up == 1:
            x = F.conv2d(x, k, padding=1)
        else:
            x = F.conv_transpose2d(x, k.transpose(0, 1), stride=2)           # [.., 2H+1, 2W+1]
            x = _fir(x, self.resample_filter, (1, 1, 1, 1), 4.0)             # -> [.., 2H, 2W]
        if noise_mode == "random":
            x = x + torch.randn(x.shape[0], 1, self.resolution, self.resolution, device=x.device, dtype=x.dtype) * self.noise_strength
        elif noise_mode == "const":
            x = x + self.noise_const * self.noise_strength
        elif noise_mode != "none":
            raise ValueError(f"noise_mode must be random / const / none, not {noise_mode!r}")
        x = F.leaky_relu(x + self.bias.view(1, -1, 1, 1), 0.2) * math.sqrt(2.0)
        return x.clamp(-self.conv_clamp, self.conv_clamp) if self.conv_clamp is not None else x


class _ToRGB(nn.Module):
    """1x1 modulated convolution without demodulation (ToRGBLayer)."""

    def __init__(self, in_channels, out_channels, w_dim, conv_clamp=256.0):
        super().__init__()
        self.conv_clamp = conv_clamp
        self.affine = _Affine(w_dim, in_channels)
        self.weight = nn.Parameter(torch.randn(out_channels, in_channels, 1, 1))
        self.bias = nn.Parameter(torch.zeros(out_channels))
        self.weight_gain = 1.0 / math.sqrt(in_channels)

    def forward(self, x, w):
        s = self.affine(w) * self.weight_gain
        y = F.conv2d(x, (self.weight * s.view(1, -1, 1, 1)).to(x.dtype)) + self.bias.view(1, -1, 1, 1)
        return y.clamp(-self.conv_clamp, self.conv_clamp) if self.conv_clamp is not None else y


class _Block(nn.Module):
    """conv0 -> conv1 -> toRGB added to the (possibly up-sampled) rgb skip: the 'skip' architecture of SynthesisBlock(NoUp)."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, up):
        super().__init__()
        self.up = up
        self.register_buffer("resample_filter", _binomial_filter())
        self.conv0 = _ModConv(in_channels, out_channels, w_dim, resolution, up=up)
        self.conv1 = _ModConv(out_channels, out_channels, w_dim, resolution)
        self.torgb = _ToRGB(out_channels, 3, w_dim)

    def forward(self, x, img, w, noise_mode="random"):
        x = self.conv0(x, w, noise_mode)
        x = self.conv1(x, w, noise_mode)
        if self.up == 2:
            img = _upsample2x(img, self.resample_filter)
        return x, img + self.torgb(x, w)


class Superresolution(nn.Module):
    """radnerf_sr.py:15-48.  forward(rgb [B,3,h,w] in [0,1]) -> [B,3,512,512] (not clamped; the caller clamps)."""

    backend = "native"   # CUDA tensors: libgfpp's sm_90a kernels; "torch": the fp32 convolutions below (always on CPU tensors)

    def __init__(self, channels=3, img_resolution=512, sr_antialias=True):
        super().__init__()
        if img_resolution != 512:
            raise NotImplementedError("the reference's SR head is 256 -> 512 only")
        self.sr_antialias = sr_antialias
        self.input_resolution = 256
        self.w_dim = 16
        self.block0 = _Block(channels, 128, self.w_dim, 256, up=1)
        self.block1 = _Block(128, 64, self.w_dim, 512, up=2)
        self.register_buffer("resample_filter", _binomial_filter())

    # ------------------------------------------------------------------ host half of the native path
    def folded_weights(self, dtype=torch.float32):
        """The six layers as plain convolutions / GEMM matrices (fp32, or `dtype`, on the parameters' device), given the constant
        latent w = 1 (radnerf_sr.py:33-34); layouts as gfpp_sr_desc (include/gfpp.h) wants them:

          conv_in_w [27,128]    block0.conv0, k = (ky*3+kx)*3 + ci                      (cross-correlation taps, padding 1)
          conv0_w   [128,1152]  block0.conv1, k = (ky*3+kx)*128 + ci
          up_w      [256,1152]  block1.conv0: y = FIR(conv_transpose2d(x, k, stride 2)) merged into four 3x3 kernels on the
                                input grid, one per output phase (py, px): row (py*2+px)*64 + co produces pixel
                                (2i+py, 2j+px).  With f = [1,3,3,1]/8 * 2 per axis (gain 4 in 2-D), u[U] = sum_a k[a] x[(U-a)/2]
                                and y[Y] = sum_t f[t] u[Y+t-1]:  K_p[o] = sum_{t,a : t-1-a = 2o-p} f[t] k[a],  o in {-1,0,1};
                                zero-extending x reproduces the padding of the reference's conv2d_resample exactly.
          conv1_w   [64,576]    block1.conv1, k = (ky*3+kx)*64 + ci
          bias[4], rgb_w[2] ([3,C]: toRGB weight * style / sqrt(C)), rgb_b[2]

        Differentiable when called with grad enabled: the native backward's gradients w.r.t. these matrices reach the conv and
        affine weights, the biases and the toRGB weights through autograd on this fold (train_ops.sr_head).
        """
        # computed on the host from CPU copies of the (small) parameters -- a few hundred tiny tensor ops that would otherwise be a
        # few hundred kernel launches per (re)pack -- and moved to the parameters' device at the end
        dev = self.block0.conv0.weight.device
        w = torch.ones(self.w_dim, dtype=dtype)
        b0, b1 = self.block0, self.block1

        def c(t):   # a tensor of its own, never the parameter itself (the model may move to another device afterwards)
            t = t.to(dtype).cpu()
            return t.clone() if torch.is_grad_enabled() else t.detach()

        def mod_w(layer):     # _ModConv.modulated_weight on the CPU copies
            s_ = torch.addmv(c(layer.affine.bias), c(layer.affine.weight) * layer.affine.weight_gain, w)
            k = c(layer.weight) * s_.view(1, -1, 1, 1)
            return k * (k.square().sum(dim=[1, 2, 3]) + 1e-8).rsqrt().view(-1, 1, 1, 1)

        k00, k01 = mod_w(b0.conv0), mod_w(b0.conv1)
        k10, k11 = mod_w(b1.conv0).double(), mod_w(b1.conv1)
        f1 = c(b1.conv0.resample_filter).double().sum(dim=0)     # separable: rows of outer(f,f)/64 sum to f/8
        f1 = f1 / f1.sum() * 2.0                                 # [1,3,3,1]/8 * 2
        O, I = k10.shape[:2]
        # per axis, M[p, o, a] = sum of the filter taps f1[t] with t - 1 - a = 2o - p (o shifted to 0..2); the phase kernels are the
        # separable product, one differentiable contraction (no in-place accumulation for autograd to replay)
        M = torch.zeros(2, 3, 3, dtype=torch.float64)
        for p in range(2):
            for t in range(4):
                for a in range(3):
                    if (p + t - 1 - a) % 2 == 0:
                        M[p, (p + t - 1 - a) // 2 + 1, a] += f1[t]
        K = torch.einsum("poa,qxb,ijab->pqijox", M, M, k10)          # [py, px, O, I, oy, ox]

        def rgb(t):
            s_ = torch.addmv(c(t.affine.bias), c(t.affine.weight) * t.affine.weight_gain, w) * t.weight_gain
            return (c(t.weight)[:, :, 0, 0] * s_.view(1, -1)).contiguous(), c(t.bias).contiguous()

        r0w, r0b = rgb(b0.torgb)
        r1w, r1b = rgb(b1.torgb)
        fw = {
            "conv_in_w": k00.permute(2, 3, 1, 0).reshape(27, 128).contiguous(),
            "conv0_w": k01.permute(0, 2, 3, 1).reshape(128, 9 * 128).contiguous(),
            "up_w": K.permute(0, 1, 2, 4, 5, 3).reshape(4 * O, 9 * I).to(dtype).contiguous(),
            "conv1_w": k11.permute(0, 2, 3, 1).reshape(64, 9 * 64).contiguous(),
            "bias": [c(b0.conv0.bias).contiguous(), c(b0.conv1.bias).contiguous(), c(b1.conv0.bias).contiguous(), c(b1.conv1.bias).contiguous()],
            "rgb_w": [r0w, r1w], "rgb_b": [r0b, r1b],
        }
        if dev.type == "cpu":
            return fw
        return {k: ([t.to(dev) for t in v] if isinstance(v, list) else v.to(dev)) for k, v in fw.items()}

    def _layers(self):
        return (self.block0.conv0, self.block0.conv1, self.block1.conv0, self.block1.conv1)

    def _native_state(self):
        """Packed weights of the native path, rebuilt when a parameter changes (in place or by load_state_dict)."""
        from . import _capi
        key = tuple((t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers()))
        st = self.__dict__.get("_native")
        if st is None or st["key"] != key:
            dev = self.block0.conv0.weight.device
            L = _capi.lib()
            with torch.no_grad():
                fw = self.folded_weights()
            d = _capi.SrDesc()
            keep = []
            for name in ("conv_in_w", "conv0_w", "up_w", "conv1_w"):
                setattr(d, name, _capi.ptr(fw[name], torch.float32))
            for i in range(4):
                d.bias[i] = _capi.ptr(fw["bias"][i], torch.float32)
            for i in range(2):
                d.rgb_w[i] = _capi.ptr(fw["rgb_w"][i], torch.float32)
                d.rgb_b[i] = _capi.ptr(fw["rgb_b"][i], torch.float32)
            packed = torch.empty(L.gfpp_sr_packed_bytes() + 1024, dtype=torch.uint8, device=dev)
            off = (-packed.data_ptr()) % 1024
            model = _capi.SrModel()
            with torch.cuda.device(dev):
                _capi.check(L.gfpp_sr_pack(ctypes.byref(d), _capi.c_void_p(packed.data_ptr() + off), packed.numel() - off,
                                           ctypes.byref(model), _capi.stream_ptr(dev)), "gfpp_sr_pack")
            strengths = [float(l.noise_strength.detach()) for l in self._layers()]       # one sync per (re)pack
            st = {"key": key, "packed": packed, "model": model, "fw": fw, "strengths": strengths, "ws": None}
            self.__dict__["_native"] = st
        return st

    @torch.no_grad()
    def forward_native(self, rgb_flat, noise_mode="random", clamp=False, out=None, frames_per_call=8, noise_planes=None, u8_out=None):
        """rgb_flat [F, R*R, 3] fp32 CUDA in [0,1] (the layout the renderer writes `rgb_map` in), R = 256 -> [F,3,2R,2R]
        through libgfpp's sm_90a kernels (4 launches per chunk of frames).  `noise_planes`: optional list of four tensors
        ([res,res] shared by all frames or [F,res,res]; None entries = no noise), already multiplied by the layers'
        noise_strength, instead of drawing them here (tests; callers that want reproducible 'random' noise).
        u8_out: optional contiguous uint8 [F,2R,2R,3] CUDA tensor that receives the video frames `(clamped rgb * 255).int()`
        straight from the last kernel (gfpp_sr_forward_video).  The result is then clamped (clamp=False is refused); `out` may be
        omitted, and without it no fp32 frame is written at all.  Returns u8_out then, else the fp32 frames."""
        from . import _capi
        R = self.input_resolution
        if not rgb_flat.is_cuda:
            raise _capi.GfppError("the native SR head needs CUDA tensors (libgfpp has no CPU path)")
        x = rgb_flat.reshape(-1, R * R, 3)
        if x.dtype != torch.float32 or not x.is_contiguous():
            x = x.float().contiguous()
        dev = x.device
        F_ = x.shape[0]
        st = self._native_state()
        L = _capi.lib()
        if u8_out is not None:
            if not clamp:
                raise ValueError("the video frames are made from the clamped image: u8_out needs clamp=True")
            if u8_out.shape != (F_, 2 * R, 2 * R, 3) or u8_out.dtype != torch.uint8 or not u8_out.is_contiguous() or u8_out.device != dev:
                raise ValueError(f"u8_out must be a contiguous uint8 [{F_},{2 * R},{2 * R},3] tensor on {dev}")
        res = out if out is not None or u8_out is not None else torch.empty(F_, 3, 2 * R, 2 * R, device=dev, dtype=torch.float32)
        if res is not None and (res.shape != (F_, 3, 2 * R, 2 * R) or res.dtype != torch.float32 or not res.is_contiguous()):
            raise ValueError(f"out must be a contiguous float32 [{F_},3,{2 * R},{2 * R}] tensor")
        if noise_mode not in ("random", "const", "none"):
            raise ValueError(f"noise_mode must be random / const / none, not {noise_mode!r}")
        layers = self._layers()
        for s0 in range(0, F_, frames_per_call):
            n = min(frames_per_call, F_ - s0)
            planes, arr = [], (_capi.c_void_p * 4)()
            per_frame = noise_mode == "random"
            if noise_planes is not None:
                per_frame = any(p is not None and p.dim() == 3 for p in noise_planes)
            for i, lay in enumerate(layers):
                p = None
                if noise_planes is not None:
                    p = noise_planes[i]
                    if p is not None:
                        p = p.to(dev, torch.float32)
                        p = (p[s0:s0 + n] if p.dim() == 3 else (p.expand(n, -1, -1) if per_frame else p)).contiguous()
                        if p.shape[-2:] != (lay.resolution, lay.resolution):
                            raise ValueError(f"noise plane {i} must be {lay.resolution}x{lay.resolution}")
                elif noise_mode != "none" and st["strengths"][i] != 0.0:
                    if noise_mode == "const":
                        p = (lay.noise_const * lay.noise_strength).float().contiguous()
                    else:
                        p = (torch.randn(n, lay.resolution, lay.resolution, device=dev) * lay.noise_strength).float().contiguous()
                planes.append(p)
                arr[i] = _capi.ptr(p, torch.float32) if p is not None else None
            need = L.gfpp_sr_workspace_bytes(n, R)
            if st["ws"] is None or st["ws"].numel() < need or st["ws"].device != dev:
                st["ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                if u8_out is None:
                    _capi.check(L.gfpp_sr_forward(ctypes.byref(st["model"]), n, R, _capi.ptr(x[s0:s0 + n], torch.float32), ctypes.byref(arr),
                                                  1 if per_frame else 0, _capi.ptr(res[s0:s0 + n], torch.float32),
                                                  1 if clamp else 0, _capi.ptr(st["ws"]), st["ws"].numel(), _capi.stream_ptr(dev)),
                                "gfpp_sr_forward")
                else:
                    _capi.check(L.gfpp_sr_forward_video(ctypes.byref(st["model"]), n, R, _capi.ptr(x[s0:s0 + n], torch.float32),
                                                        ctypes.byref(arr), 1 if per_frame else 0,
                                                        None if res is None else _capi.ptr(res[s0:s0 + n], torch.float32),
                                                        _capi.ptr(u8_out[s0:s0 + n], torch.uint8), _capi.ptr(st["ws"]), st["ws"].numel(),
                                                        _capi.stream_ptr(dev)), "gfpp_sr_forward_video")
        return res if u8_out is None else u8_out

    def forward(self, rgb, noise_mode="random"):
        if rgb.is_cuda and self.backend == "native" and rgb.shape[-2:] == (self.input_resolution, self.input_resolution):
            x = rgb.float().permute(0, 2, 3, 1).reshape(rgb.shape[0], -1, 3)
            if torch.is_grad_enabled() and (rgb.requires_grad or any(p.requires_grad for p in self.parameters())):
                from . import train_ops
                return train_ops.sr_head(self, x, noise_mode)
            return self.forward_native(x, noise_mode=noise_mode)
        x = rgb.float()
        if x.shape[-1] < self.input_resolution:
            x = F.interpolate(x, size=(self.input_resolution, self.input_resolution), mode="bilinear", align_corners=False,
                              antialias=self.sr_antialias)
        if x.shape[-2:] != (self.input_resolution, self.input_resolution):
            raise ValueError(f"SR input must be at most {self.input_resolution}x{self.input_resolution}, got {tuple(rgb.shape)}")
        w = torch.ones(self.w_dim, dtype=x.dtype, device=x.device)
        feat, img = self.block0(x, x, w, noise_mode)
        _, img = self.block1(feat, img, w, noise_mode)
        return img
