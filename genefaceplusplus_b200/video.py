"""Planar I420 (yuv420p) video frames: the format video encoders take, at half the bytes of interleaved RGB.

`rgb_u8_to_i420` converts the renderer's uint8 RGB frames on the GPU (libgfpp's gfpp_rgb_u8_to_i420, include/gfpp.h section N):
BT.601 limited range in integer arithmetic, chroma the 2x2 box average (centre siting).  Each frame is Y [H,W], U [H/2,W/2],
V [H/2,W/2] back to back, and frames follow one another, so a chunk of frames is one write to
`ffmpeg -f rawvideo -pix_fmt yuv420p -s WxH -r 25 -i - ... -colorspace smpte170m -color_range tv`.  The bytes are not those of
ffmpeg's own RGB -> yuv420p conversion (swscale), whose rounding and chroma filter differ.

`i420_reference` restates the conversion in numpy, byte for byte: the host reference of the tests and of tools/yuv_bench.py.
"""
import numpy as np
import torch

from . import _capi


def i420_frame_bytes(H, W):
    """Bytes of one H x W yuv420p frame: H*W luma + two (H/2)*(W/2) chroma planes."""
    return H * W * 3 // 2


def check_i420_size(H, W):
    """yuv420p (and libx264) need even frame sizes: ValueError otherwise."""
    if H <= 0 or W <= 0 or H % 2 or W % 2:
        raise ValueError(f"I420 frames need an even, non-zero height and width (4:2:0 chroma is subsampled 2x2), not {H}x{W}")


def rgb_u8_to_i420(rgb, H, W, out=None):
    """rgb: contiguous uint8 CUDA tensor of F frames of H x W interleaved RGB ([F,H,W,3] or [F,H*W,3]) -> uint8 [F, H*W*3/2]
    I420 frames, written into `out` (optional contiguous uint8 CUDA tensor of that size) on the current stream."""
    check_i420_size(H, W)
    if rgb.dtype != torch.uint8 or rgb.numel() % (H * W * 3) or rgb.numel() == 0:
        raise ValueError(f"rgb must be uint8 frames of {H}x{W}x3 bytes")
    F = rgb.numel() // (H * W * 3)
    fb = i420_frame_bytes(H, W)
    if out is None:
        out = torch.empty(F, fb, dtype=torch.uint8, device=rgb.device)
    if out.dtype != torch.uint8 or out.numel() != F * fb or not out.is_contiguous() or out.device != rgb.device:
        raise ValueError(f"out must be a contiguous uint8 [{F},{fb}] tensor on {rgb.device}")
    L = _capi.lib()
    src, dst = _capi.ptr(rgb, torch.uint8), _capi.ptr(out, torch.uint8)
    with torch.cuda.device(rgb.device):
        _capi.check(L.gfpp_rgb_u8_to_i420(src, F, H, W, dst, _capi.stream_ptr(rgb.device)), "gfpp_rgb_u8_to_i420")
    return out.view(F, fb)


def i420_reference(rgb):
    """numpy restatement of gfpp_rgb_u8_to_i420: uint8 [F,H,W,3] -> uint8 [F, H*W*3/2]."""
    F, H, W, _ = rgb.shape
    check_i420_size(H, W)
    x = rgb.astype(np.int32)
    y = ((66 * x[..., 0] + 129 * x[..., 1] + 25 * x[..., 2] + 128) >> 8) + 16
    m = (x.reshape(F, H // 2, 2, W // 2, 2, 3).sum(axis=(2, 4)) + 2) >> 2          # the 2x2 blocks' rounded means
    r, g, b = m[..., 0], m[..., 1], m[..., 2]
    u = ((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128                              # numpy's >> on int32 is arithmetic
    v = ((112 * r - 94 * g - 18 * b + 128) >> 8) + 128
    return np.concatenate([y.reshape(F, -1), u.reshape(F, -1), v.reshape(F, -1)], axis=1).astype(np.uint8)


def frame_scratch(model, shape):
    """A uint8 view of `shape` on the model's device, from one buffer the model keeps between calls: the RGB frames of a chunk on
    their way to I420.  Grown to the largest chunk seen; used stream-ordered on the current stream."""
    dev = model.density_bitfield.device
    n = int(np.prod(shape))
    buf = model.__dict__.get("_i420_scratch")
    if buf is None or buf.numel() < n or buf.device != dev:
        buf = torch.empty(n, dtype=torch.uint8, device=dev)
        model.__dict__["_i420_scratch"] = buf
    return buf[:n].view(shape)
