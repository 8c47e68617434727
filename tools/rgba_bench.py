"""tools/rgba_bench.py -- what the alpha-matte frames cost on one GPU: 50-frame clips of the bench scene (512x512 head + torso,
density_scale 8, max_steps 16, T_thresh 0.01, random-init May weights), one libgfpp call per clip, in three arms:

    u8          render_clip(as_uint8=True, bg_color=bg)   video frames over the background   3 B/pixel written by k_epilogue
    rgba        render_clip(as_rgba=True)                 premultiplied RGBA matte            4 B/pixel
    rgba_alpha  render_frames(rgba_out=, alpha_out=)      RGBA + the fp32 coverage map        8 B/pixel

Arms alternate within every repetition after one warm-up call of each; a call is timed with CUDA events and ends in a synchronise.
A second alternating pass with libgfpp's event profile on (gfpp_profile_enable) reads the epilogue kernel's own time per call.
Medians over the repetitions are reported, with min and max.  Prints JSON lines, the device name and power limit first.

    python tools/rgba_bench.py [--frames 50] [--reps 30] [--precision fp16] [--out out/rgba_bench.jsonl]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import _capi  # noqa: E402
from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRFTorso  # noqa: E402


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except Exception as e:   # the numbers are still printed; the missing context is said so
        info["power_limit"] = f"unknown ({type(e).__name__})"
    return info


def ms(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def epilogue_ms(fn):
    L = _capi.lib()
    fn()
    buf = (ctypes.c_float * 4)()
    _capi.check(L.gfpp_profile_read(buf), "gfpp_profile_read")
    return buf[2]


def alternate(arms, reps, timer):
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(timer(fn))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--precision", default="fp16", choices=["fp32", "fp16", "robust", "bf16x3", "bf16"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rgba_bench needs a CUDA device (there is nothing to measure on the CPU)")
    T, H = a.frames, 512
    N = H * H
    sc = scn.Scene(H=H, W=H, T=T, torso=True, density_scale=8.0)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m.mlp_precision = a.precision
    m = m.cuda().eval()
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    pose6 = scn.convert_poses(poses.cpu()).cuda()
    feat = m.cal_cond_feat_clip(sc.cond.cuda())[:T]
    bg_color, bg_coords = sc.bg_color.cuda(), sc.bg_coords.cuda()
    u8 = torch.empty(T, N, 3, dtype=torch.uint8, device="cuda")
    rgba = torch.empty(T, N, 4, dtype=torch.uint8, device="cuda")
    alpha = torch.empty(T, N, device="cuda")
    clip = dict(cond_feat=feat, bg_coords=bg_coords, pose6=pose6, T_thresh=sc.T_thresh, frames_per_call=T)
    arms = {
        "u8": lambda: m.render_clip(poses, sc.intrinsics, H, H, bg_color=bg_color, out=u8, as_uint8=True, **clip),
        "rgba": lambda: m.render_clip(poses, sc.intrinsics, H, H, out=rgba, as_rgba=True, **clip),
        "rgba_alpha": lambda: m.render_frames(feat, poses_c2w=poses, intrinsics=sc.intrinsics, H=H, W=H, pose6=pose6, bg_coords=bg_coords,
                                              dt_gamma=sc.hparams["dt_gamma"], max_steps=sc.hparams["max_steps"], T_thresh=sc.T_thresh,
                                              want_torso_maps=False, want_aux=False, rgba_out=rgba, alpha_out=alpha),
    }
    bytes_per_pixel = {"u8": 3, "rgba": 4, "rgba_alpha": 8}
    lines = [{"what": "context", "frames_per_call": T, "size": H, "reps": a.reps, "precision": a.precision, **device_info()}]
    print(json.dumps(lines[0]), flush=True)
    calls = alternate(arms, a.reps, ms)
    L = _capi.lib()
    L.gfpp_profile_enable(1)
    try:
        epi = alternate(arms, a.reps, epilogue_ms)
    finally:
        L.gfpp_profile_enable(0)
    base = sorted(calls["u8"])[a.reps // 2]
    for k in arms:
        c, e = sorted(calls[k]), sorted(epi[k])
        med = c[a.reps // 2]
        lines.append({"arm": k, "epilogue_bytes_written_per_pixel": bytes_per_pixel[k], "ms_per_call": med, "min_ms": c[0], "max_ms": c[-1],
                      "frames_per_s": 1000.0 * T / med, "vs_u8": med / base, "epilogue_ms": e[a.reps // 2], "epilogue_min_ms": e[0],
                      "epilogue_max_ms": e[-1]})
        print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
