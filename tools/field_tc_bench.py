"""Time the head field of one training step in both libgfpp arithmetics beside the eager paths, on the bench scene's ray batch: one
256x256 frame (65 536 rays), max_steps 16 -- the shape of tools/train_step_bench.py.

    python tools/field_tc_bench.py [--reps 9] [--warmup 3] [--profile DIR]

Legs, alternated round by round in one process (one call of every leg per round, so drift of the card's clocks reaches all legs
alike); each figure is the median of its CUDA-event timings after the warm-up rounds:
  gfpp_fp32   RADNeRF.forward with train_precision "fp32" (gfpp.h section G): forward; forward + backward; the whole render() step
  gfpp_fp16   the same with train_precision "fp16" (section J: fp16 wgmma operands, fp32 accumulation)
  eager_fp32  the restatement of radnerf.py:108-141 in eager PyTorch (F.linear, TF32 off) over libgfpp's per-op grid kernels
  eager_amp   the same under fp16 autocast (the reference's amp: true arithmetic)
Prints one JSON line: the card's name and power limit read in the same run, the point count, the algorithmic GFLOP from the shapes,
the times, the whole-call TFLOP/s of both libgfpp legs (algorithmic FLOP over the time of the whole forward + backward call,
relayout, gathers and scatters included: not a kernel's rate), and the largest relative difference between the two arithmetics'
gradients on the timed inputs.  --profile DIR runs torch.profiler (CUDA activities) over three forward + backward calls per libgfpp
arithmetic in a separate pass after the timing and writes DIR/field_tc_kernels.json with the mean time per kernel.
Needs a GPU: there is no CPU fallback.
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
from genefaceplusplus_b200.renderer import RADNeRF  # noqa: E402
from oracle import field_train as ft  # noqa: E402


def flops_per_point(A):
    """Forward multiply-adds x 2 of the eight layers; the backward needs the input and the weight gradient of each: twice that."""
    macs = 96 * 128 + 128 * 128 + 128 * A + 64 * 128 + 128 * 128 + 128 * 129 + 148 * 128 + 128 * 3
    return 2 * macs, 4 * macs


def time_alternated(legs, reps, warmup):
    """legs: name -> callable.  Returns name -> median ms over `reps` rounds; every round runs each leg once, in order."""
    ts = {k: [] for k in legs}
    for r in range(warmup + reps):
        for k, fn in legs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if r >= warmup:
                ts[k].append(a.elapsed_time(b))
    return {k: sorted(v)[len(v) // 2] for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("field_tc_bench measures on the GPU: no CUDA device found")
    if args.reps < 7 or args.warmup < 3:
        raise SystemExit("at least 7 timed rounds after at least 3 warm-up rounds")
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
    g = torch.Generator(device="cuda").manual_seed(3)
    gs, gc = torch.randn(M, device="cuda", generator=g), torch.randn(M, 3, device="cuda", generator=g)
    ga = torch.randn(M, m.ambient_coord_dim, device="cuda", generator=g)
    P = {k: p for k, p in m.named_parameters() if k in ft.TRAINABLE}
    render_in = [fi[k].cuda() for k in ("rays_o", "rays_d", "cond", "bg_color")]

    def loss_of(f):
        s, c, a = f
        return (s * gs).sum() + (c * gc).sum() + (a * ga).sum()

    def gfpp_fwd(precision):
        m.train_precision = precision
        with torch.no_grad():
            m.forward(xyzs, dirs, cond, code)

    def gfpp_fb(precision):
        m.train_precision = precision
        m.zero_grad(set_to_none=True)
        loss_of(m.forward(xyzs, dirs, cond, code)).backward()

    def eager_fwd(amp):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            ft.eager_field(m, P, xyzs, dirs, cond, code, train_ops.grid_encode)

    def eager_fb(amp):
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            out = ft.eager_field(m, P, xyzs, dirs, cond, code, train_ops.grid_encode)
        loss_of(tuple(t.float() for t in out)).backward()

    def render_step(precision):
        m.train_precision = precision
        m.train()
        m.zero_grad(set_to_none=True)
        res = m.render(render_in[0], render_in[1], render_in[2], None, None, bg_color=render_in[3], max_steps=16)
        (res["rgb_map"].square().mean() + res["ambient"].mean()).backward()
        m.eval()

    legs = {}
    for name, prec in (("gfpp_fp32", "fp32"), ("gfpp_fp16", "fp16")):
        legs[f"{name}_forward_ms"] = lambda p=prec: gfpp_fwd(p)
        legs[f"{name}_fwd_bwd_ms"] = lambda p=prec: gfpp_fb(p)
        legs[f"{name}_render_step_ms"] = lambda p=prec: render_step(p)
    for name, amp in (("eager_fp32", False), ("eager_amp", True)):
        legs[f"{name}_forward_ms"] = lambda a=amp: eager_fwd(a)
        legs[f"{name}_fwd_bwd_ms"] = lambda a=amp: eager_fb(a)
    ms = time_alternated(legs, args.reps, args.warmup)

    grads = {}
    for prec in ("fp32", "fp16"):
        gfpp_fb(prec)
        grads[prec] = {k: p.grad.detach().clone() for k, p in P.items()}
    grad_diff = max(((grads["fp16"][k] - grads["fp32"][k]).abs().max() / grads["fp32"][k].abs().max()).item() for k in P)

    fwd, bwd = flops_per_point(m.ambient_coord_dim)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
    power = q.stdout.strip() if q.returncode == 0 else f"unavailable ({q.stderr.strip()})"
    out = {"tool": "field_tc_bench", "gpu": torch.cuda.get_device_name(0), "power_limit": power, "rays": rays_o.shape[0], "max_steps": 16,
           "points": M, "fwd_gflop": round(fwd * M / 1e9, 3), "fwd_bwd_gflop": round((fwd + bwd) * M / 1e9, 3),
           "median_of": args.reps, "warmup": args.warmup}
    out.update({k: round(v, 4) for k, v in ms.items()})
    for name in ("gfpp_fp32", "gfpp_fp16"):
        out[f"{name}_fwd_bwd_whole_call_tflops"] = round((fwd + bwd) * M / (ms[f"{name}_fwd_bwd_ms"] * 1e-3) / 1e12, 2)
    out["fp16_vs_fp32_max_rel_grad_diff"] = round(grad_diff, 6)
    print(json.dumps(out))

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        table = {}
        for prec in ("fp32", "fp16"):
            gfpp_fb(prec)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    gfpp_fb(prec)
                torch.cuda.synchronize()
            rows = [(e.key, e.device_time_total / 3e3, e.count // 3) for e in prof.key_averages() if e.device_time_total > 0]
            table[prec] = [{"kernel": k, "ms_per_call": round(t, 4), "launches_per_call": n} for k, t, n in sorted(rows, key=lambda r: -r[1])]
        with open(os.path.join(args.profile, "field_tc_kernels.json"), "w") as f:
            json.dump({"gpu": out["gpu"], "power_limit": power, "points": M, "forward_plus_backward": table}, f, indent=1)


if __name__ == "__main__":
    main()
