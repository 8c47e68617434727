"""Time one training step's head field on the bench scene's ray batch: one 256x256 frame (65 536 rays), max_steps 16.

    python tools/train_step_bench.py [--reps 7] [--warmup 3]

Legs, each a median of CUDA-event timings after warm-up:
  gfpp      RADNeRF.forward (libgfpp, gfpp.h section G): forward; forward + backward; the whole differentiable render() step
            (marching, field, compositing, loss, backward)
  eager     the fp32 restatement of radnerf.py:108-141 in eager PyTorch (F.linear with TF32 off) over libgfpp's per-op grid kernels
  amp       the same under fp16 autocast (the reference's amp: true arithmetic)
  ref       the eager fp32 restatement over the reference's OWN compiled grid-encoder kernels (oracle/_ref/_gridencoder, built where the
            reference sources exist); reported as unavailable when they are not present
Prints one JSON line with the card name and power limit read in the same run, the point count and the algorithmic GFLOP computed from
the shapes.  The backward runs FIELD_CTAS = 132 persistent CTAs at one per SM (an H100 SXM's SM count); a part with fewer SMs runs
them as a second, partly filled wave.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200 import train_ops  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRF  # noqa: E402
from oracle import field_train as ft  # noqa: E402


class _RefGridEncode(torch.autograd.Function):
    """grid.py:24-88 over the reference's own compiled `_gridencoder` (fp32)."""

    @staticmethod
    def forward(ctx, inputs, embeddings, offsets, per_level_scale, base_resolution, calc_grad_inputs, gridtype, align_corners, interp):
        import numpy as np
        from oracle import gpu_ref_ops
        mod = gpu_ref_ops._load("_gridencoder")
        inputs, embeddings = inputs.float().contiguous(), embeddings.float().contiguous()
        B, D = inputs.shape
        L, C = offsets.shape[0] - 1, embeddings.shape[1]
        S = float(np.log2(per_level_scale))
        out = torch.empty(L, B, C, device=inputs.device)
        dy_dx = torch.empty(B, L * D * C, device=inputs.device) if calc_grad_inputs else None
        mod.grid_encode_forward(inputs, embeddings, offsets, out, B, D, C, L, S, base_resolution, dy_dx, gridtype, align_corners, interp)
        ctx.save_for_backward(inputs, embeddings, offsets, dy_dx)
        ctx.dims = (B, D, C, L, S, base_resolution, gridtype, interp, align_corners, mod)
        return out.permute(1, 0, 2).reshape(B, L * C)

    @staticmethod
    def backward(ctx, grad):
        inputs, embeddings, offsets, dy_dx = ctx.saved_tensors
        B, D, C, L, S, H, gridtype, interp, align_corners, mod = ctx.dims
        grad = grad.float().view(B, L, C).permute(1, 0, 2).contiguous()
        ge = torch.zeros_like(embeddings)
        gi = torch.zeros_like(inputs) if dy_dx is not None else None
        mod.grid_encode_backward(grad, inputs, embeddings, offsets, ge, B, D, C, L, S, H, dy_dx, gi, gridtype, align_corners, interp)
        return gi, ge, None, None, None, None, None, None, None


def _ref_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "_gridencoder", "_gridencoder.so"))


def flops_per_point(A):
    """Forward multiply-adds x 2 of the eight layers; the backward needs the input and the weight gradient of each: twice that."""
    macs = 96 * 128 + 128 * 128 + 128 * A + 64 * 128 + 128 * 128 + 128 * 129 + 148 * 128 + 128 * 3
    return 2 * macs, 4 * macs


def timeit(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool measures on the GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    sc = scn.Scene(H=256, W=256, T=2, torso=False, density_scale=8.0)
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m = m.cuda()
    fi = sc.frame_inputs(0)
    rays_o, rays_d = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
    nears, fars = train_ops.near_far_from_aabb(rays_o, rays_d, m.aabb_train, m.min_near)
    xyzs, dirs, deltas, rays = train_ops.march_rays_train(rays_o, rays_d, m.bound, m.density_bitfield, m.cascade, m.grid_size, nears, fars,
                                                          None, 0, False, 128, False, 0, 16)
    M = xyzs.shape[0]
    cond = m.cal_cond_feat(fi["cond"].cuda()).detach().reshape(1, -1)
    code = m.individual_embeddings[0]
    gs, gc, ga = torch.randn(M, device="cuda"), torch.randn(M, 3, device="cuda"), torch.randn(M, m.ambient_coord_dim, device="cuda")
    P = {k: p for k, p in m.named_parameters() if k in ft.TRAINABLE}

    def loss_of(f):
        s, c, a = f
        return (s * gs).sum() + (c * gc).sum() + (a * ga).sum()

    def gfpp_fwd():
        with torch.no_grad():
            m.forward(xyzs, dirs, cond, code)

    def gfpp_fb():
        m.zero_grad(set_to_none=True)
        loss_of(m.forward(xyzs, dirs, cond, code)).backward()

    def eager_fwd(amp=False, ge=train_ops.grid_encode):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            ft.eager_field(m, P, xyzs, dirs, cond, code, ge)

    def eager_fb(amp=False, ge=train_ops.grid_encode):
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            out = ft.eager_field(m, P, xyzs, dirs, cond, code, ge)
        loss_of(tuple(t.float() for t in out)).backward()

    def render_step():
        m.train()
        m.zero_grad(set_to_none=True)
        res = m.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), None, None, bg_color=fi["bg_color"].cuda(), max_steps=16)
        (res["rgb_map"].square().mean() + res["ambient"].mean()).backward()
        m.eval()

    r, w = args.reps, args.warmup
    ms = {
        "gfpp_forward_ms": timeit(gfpp_fwd, r, w), "gfpp_fwd_bwd_ms": timeit(gfpp_fb, r, w), "gfpp_render_step_ms": timeit(render_step, r, w),
        "eager_fp32_forward_ms": timeit(eager_fwd, r, w), "eager_fp32_fwd_bwd_ms": timeit(eager_fb, r, w),
        "eager_amp_forward_ms": timeit(lambda: eager_fwd(True), r, w), "eager_amp_fwd_bwd_ms": timeit(lambda: eager_fb(True), r, w),
    }
    if _ref_available():
        ms["ref_kernels_fp32_forward_ms"] = timeit(lambda: eager_fwd(False, _RefGridEncode.apply), r, w)
        ms["ref_kernels_fp32_fwd_bwd_ms"] = timeit(lambda: eager_fb(False, _RefGridEncode.apply), r, w)
    fwd, bwd = flops_per_point(m.ambient_coord_dim)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip()
    except Exception as e:   # reported, not fatal
        power = f"unavailable ({e})"
    out = {"tool": "train_step_bench", "gpu": torch.cuda.get_device_name(0), "power_limit": power, "rays": rays_o.shape[0], "max_steps": 16,
           "points": M, "fwd_flop_per_point": fwd, "bwd_flop_per_point": bwd, "fwd_gflop": round(fwd * M / 1e9, 3),
           "fwd_bwd_gflop": round((fwd + bwd) * M / 1e9, 3), "median_of": r}
    out.update({k: round(v, 4) for k, v in ms.items()})
    if not _ref_available():
        out["ref_kernels"] = "oracle/_ref/_gridencoder not present (built where the reference sources exist)"
    out["gfpp_fwd_bwd_tflops"] = round((fwd + bwd) * M / (ms["gfpp_fwd_bwd_ms"] * 1e-3) / 1e12, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
