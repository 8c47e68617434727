"""tools/torso_train_bench.py -- timings of the trainable torso field (gfpp.h section H) and of the torso training step, one JSON line.

    python tools/torso_train_bench.py [--iters 20] [--warmup 5]

CUDA events around each leg, median over --iters after --warmup, on the synthetic May torso scene (oracle/torso_train.golden_scene):
  * forward_torso in training mode, forward and forward + backward, at 65 536 and 262 144 points (the fused libgfpp kernels);
  * the same in eager PyTorch, fp32 (F.linear over train_ops.grid_encode with input gradients; TF32 off) and under fp16 autocast;
  * the same eager field over the reference's own grid kernels (oracle/_ref), when they were built;
  * the whole torso training step (oracle/torso_train.gfpp_train_step, the README recipe) at 65 536 rays, split into the head part
    (marching, head field under no_grad, compositing) and the torso part (mask, forward_torso, composite, loss, backward);
  * that step and its head part with the head as one RADNeRF.frozen_head call against the composed head, in fp32 and fp16,
    the legs alternating in one process (--rounds).
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200 import train_ops  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRFTorso  # noqa: E402
from oracle import torso_train as tt  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return round(ts[len(ts) // 2], 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the frozen_head / composed legs")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    sc = tt.golden_scene()
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale, m.mlp_precision = tt.GOLDEN_DS, "fp32"
    m = m.cuda().train()
    P = {k: p for k, p in m.named_parameters() if k in tt.TRAINABLE}
    pose6 = sc.frame_inputs(1)["poses"].cuda()
    idx = torch.tensor([1], device="cuda")
    out = {}

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train_step_bench   # its autograd Function over the reference's own compiled grid encoder
    ref_encode = train_step_bench._RefGridEncode.apply if train_step_bench._ref_available() else None
    if ref_encode is None:
        out["reference_grid_kernels"] = "oracle/_ref/_gridencoder not present (built where the reference sources exist)"

    def eager(x, poses, c, enc=train_ops.grid_encode):
        return tt.eager_torso(m, P, x, poses, c, enc)

    for M in (65536, 262144):
        x = (torch.rand(M, 2, generator=torch.Generator().manual_seed(M)) * 2 - 1).cuda()
        legs = {"fused": lambda x, p, c: m.forward_torso(x, p, c), "eager_fp32": eager}
        legs["eager_fp16_autocast"] = lambda x, p, c: _autocast(eager, x, p, c)
        if ref_encode is not None:
            legs["eager_ref_grid_kernels"] = lambda x, p, c: eager(x, p, c, ref_encode)
        for name, f in legs.items():
            def fwd():
                with torch.no_grad():
                    f(x, pose6, m.torso_individual_codes[idx])

            def fwd_bwd():
                m.zero_grad(set_to_none=True)
                a, c, d = f(x, pose6, m.torso_individual_codes[idx])
                (a.float().sum() + c.float().sum() + d.float().sum()).backward()
            out[f"{name}.fwd_ms@{M}"] = timed(fwd, args.iters, args.warmup)
            out[f"{name}.fwd_bwd_ms@{M}"] = timed(fwd_bwd, args.iters, args.warmup)

    # the torso training step at 65 536 rays (256 x 256), head part and torso part
    big = scn.Scene(H=256, W=256, T=4, torso=True, density_scale=tt.GOLDEN_DS)
    fi = big.frame_inputs(1)
    ro, rd, cond = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3), fi["cond"].cuda()
    bgc, bgcol = fi["bg_coords"].cuda().reshape(-1, 2), fi["bg_color"].cuda().reshape(-1, 3)
    gt = torch.rand(ro.shape[0], 3, device="cuda")
    holder = {}

    def head_part():
        holder["res"] = tt.gfpp_train_step(m, ro, rd, cond, bgc, pose6, idx, bgcol, 16, torso_field=_no_torso)

    def step():
        m.zero_grad(set_to_none=True)
        res = tt.gfpp_train_step(m, ro, rd, cond, bgc, pose6, idx, bgcol, 16)
        tt.task_loss(res, gt, tt.LAMBDA_WEIGHTS_ENTROPY).backward()
        holder["pixels"] = int(res["deform"].shape[0])

    out["step_ms@65536"] = timed(step, args.iters, args.warmup)
    out["step.head_part_ms@65536"] = timed(head_part, args.iters, args.warmup)
    out["step.torso_part_ms@65536"] = round(out["step_ms@65536"] - out["step.head_part_ms@65536"], 4)
    out["step.torso_pixels"] = holder["pixels"]

    # the same step with its no-grad head block as one RADNeRF.frozen_head call (gfpp.h section K), against the composed head, in
    # fp32 and fp16 (composed: the training field with train_precision "fp16"; frozen_head: mlp_precision "fp16").  The legs
    # alternate, --rounds times, in this process; each number is the median over the rounds of the per-round medians.
    def with_precision(prec, frozen, fn):
        def run():
            m.mlp_precision, m.train_precision = (prec, "fp32") if frozen else ("fp32", prec)
            fn(frozen)
        return run

    def head_only(frozen):
        f = frozen_train_step if frozen else tt.gfpp_train_step
        holder["res"] = f(m, ro, rd, cond, bgc, pose6, idx, bgcol, 16, torso_field=_no_torso)

    def full_step(frozen):
        m.zero_grad(set_to_none=True)
        res = (frozen_train_step if frozen else tt.gfpp_train_step)(m, ro, rd, cond, bgc, pose6, idx, bgcol, 16)
        tt.task_loss(res, gt, tt.LAMBDA_WEIGHTS_ENTROPY).backward()

    legs = {}
    for prec in ("fp32", "fp16"):
        for frozen in (False, True):
            name = f"{'frozen_head' if frozen else 'composed'}.{prec}"
            legs[f"{name}.step_ms@65536"] = with_precision(prec, frozen, full_step)
            legs[f"{name}.head_part_ms@65536"] = with_precision(prec, frozen, head_only)
    rounds = {k: [] for k in legs}
    for _ in range(args.rounds):
        for k, f in legs.items():
            rounds[k].append(timed(f, args.iters, args.warmup))
    m.mlp_precision, m.train_precision = "fp32", "fp32"
    for k, v in rounds.items():
        out[k] = sorted(v)[len(v) // 2]
    for prec in ("fp32", "fp16"):
        c, f = out[f"composed.{prec}.head_part_ms@65536"], out[f"frozen_head.{prec}.head_part_ms@65536"]
        out[f"frozen_head.{prec}.head_part_speedup"] = round(c / f, 3)
    name, power = card()
    print(json.dumps({"tool": "torso_train_bench", "gpu": name, "power_limit": power, "iters": args.iters, "warmup": args.warmup, **out}))


def frozen_train_step(model, rays_o, rays_d, cond, bg_coords, poses, index, bg_color, max_steps, torso_field=None):
    """oracle/torso_train.gfpp_train_step with its no-grad head block replaced by one RADNeRF.frozen_head call."""
    rays_o, rays_d, bg_coords = rays_o.reshape(-1, 3), rays_d.reshape(-1, 3), bg_coords.reshape(-1, 2)
    with torch.no_grad():
        cond_feat = model.cal_cond_feat(cond)
    weights_sum, image = model.frozen_head(rays_o, rays_d, cond_feat, model.individual_embeddings[index], max_steps=max_steps)
    mask = model.torso_mask(bg_coords)
    N = rays_o.shape[0]
    torso_alpha = torch.zeros(N, 1, device=rays_o.device)
    torso_color = torch.zeros(N, 3, device=rays_o.device)
    alpha, color, deform = (torso_field or model.forward_torso)(bg_coords[mask], poses, model.torso_individual_codes[index])
    torso_alpha[mask] = alpha
    torso_color[mask] = color
    bg = torso_color * torso_alpha + bg_color.reshape(-1, 3) * (1 - torso_alpha)
    rgb = (image + (1 - weights_sum).unsqueeze(-1) * bg).clamp(0, 1)
    return {"torso_alpha_map": torso_alpha, "torso_rgb_map": bg, "rgb_map": rgb, "weights_sum": weights_sum, "deform": deform}


def _autocast(f, x, p, c):
    with torch.autocast("cuda", dtype=torch.float16):
        return f(x, p, c)


def _no_torso(x, poses, c):
    """The head part alone: the step with an empty torso field (no torso MLP, no backward)."""
    n = x.shape[0]
    z = torch.zeros(n, 1, device=x.device)
    return z, torch.zeros(n, 3, device=x.device), torch.zeros(n, 2, device=x.device)


if __name__ == "__main__":
    main()
