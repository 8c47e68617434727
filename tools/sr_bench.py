"""tools/sr_bench.py -- measurement of the SR-variant paths (SURVEY 8(f) rank 3) on one H100: frames/s of the clip APIs with every
stage in libgfpp (head field at 256x256 with in-kernel rays, torso-SR field, SR head on wgmma) beside the same clip with the SR
head / torso field as host-side PyTorch (cuDNN), and the stages timed alone with CUDA events.  Prints JSON lines.

    python tools/sr_bench.py [--frames 64] [--reps 5] [--out gpurun_out/sr_bench.jsonl]

Tensor-side roofline of the SR head: ALGORITHMIC flops per frame = 2 * (256^2 * (27*128 + 1152*128 + 1152*64) + 512^2 * (576*64 + 64*3)
+ 256^2 * 128*3) = 49.0 GFLOP (the transposed convolution counted as the reference computes it, not with the 4x of the merged
phase kernels), against the measured dense bf16 peak of MEASURED_PEAKS.json."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.config import may_hparams  # noqa: E402

SR_FLOPS = 2.0 * (256 ** 2 * (27 * 128 + 1152 * 128 + 1152 * 64 + 128 * 3) + 512 ** 2 * (576 * 64 + 64 * 3))


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ms = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
    return ms[len(ms) // 2]


def measure(frames=64, reps=5):
    """-> list of result dicts (see the module docstring); importable by bench.py for its `sr_variants` object."""
    class a:   # noqa: N801
        pass
    a.frames, a.reps = frames, reps
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR, RADNeRFwithSR
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))
    T = a.frames
    lines = []
    ov = {"with_sr": True, "add_eye_blink_cond": True, "eye_blink_dim": 4, "smo_win_size": 3}
    sc = scn.Scene(H=256, W=256, T=T, torso=True, density_scale=8.0)
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    eye = torch.full((T,), 0.37)
    # ---- head-SR model
    hp = may_hparams(**ov)
    m = RADNeRFwithSR(hp)
    m.load_state_dict(scn.make_head_sr_state(hp), strict=True)
    m.density_scale = 8.0
    m.mlp_precision = "fp16"
    m = m.cuda().eval()
    kw = dict(cond_seq=sc.cond.cuda(), bg_color=sc.bg_color.cuda(), eye_area_percent=eye, max_steps=16, T_thresh=sc.T_thresh, sr_noise_mode="const")
    for backend in ("native", "torch"):
        m.sr_net.backend = backend
        ms = timed(lambda: m.render_clip(poses, sc.intrinsics, 256, 256, **kw), a.reps)
        lines.append({"what": "head-SR clip (NeRF 256x256 fp16 + SR head)", "sr_backend": backend, "frames": T, "ms": ms, "fps": T / ms * 1e3})
    # SR head alone on resident frames
    rgb = torch.rand(T, 256 * 256, 3, device="cuda")
    out = torch.empty(T, 3, 512, 512, device="cuda")
    m.sr_net.backend = "native"
    ms = timed(lambda: m.sr_net.forward_native(rgb, noise_mode="const", clamp=True, out=out), a.reps)
    lines.append({"what": "SR head alone, libgfpp (4 launches per 8 frames)", "frames": T, "ms": ms, "ms_per_frame": ms / T, "tflops_algorithmic": SR_FLOPS * T / ms / 1e9,
                  "tensor_frac_of_sustained_bf16_peak": SR_FLOPS * T / ms / 1e9 / peak_tf})
    m.sr_net.backend = "torch"
    x = rgb.view(T, 256, 256, 3).permute(0, 3, 1, 2)
    with torch.no_grad():
        ms = timed(lambda: [m.sr_net(x[s:s + 8], noise_mode="const") for s in range(0, T, 8)], a.reps)
    lines.append({"what": "SR head alone, host-side PyTorch fp32 convolutions (cuDNN)", "frames": T, "ms": ms, "ms_per_frame": ms / T})
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        ms = timed(lambda: [m.sr_net(x[s:s + 8], noise_mode="const") for s in range(0, T, 8)], a.reps)
    lines.append({"what": "SR head alone, host-side PyTorch under fp16 autocast (cuDNN; how the reference runs these blocks)", "frames": T, "ms": ms, "ms_per_frame": ms / T})
    del m
    # ---- torso-SR model
    hp = may_hparams(**{**ov, "torso_head_aware": True})
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = 8.0
    m.mlp_precision = "fp16"
    m = m.cuda().eval()
    lm = scn.lm68_sequence(T).cuda()
    kw = dict(cond_seq=sc.cond.cuda(), bg_color=sc.bg_color.cuda(), bg_coords=sc.bg_coords.cuda(), lm68_seq=lm, eye_area_percent=eye, max_steps=16,
              T_thresh=sc.T_thresh, sr_noise_mode="const")
    m.torso_backend, m.sr_net.backend = "native", "native"
    ms = timed(lambda: m.render_clip(poses, sc.intrinsics, 256, 256, **kw), a.reps)
    lines.append({"what": "torso-SR clip, every stage in libgfpp", "frames": T, "ms": ms, "fps": T / ms * 1e3})
    img = torch.rand(T, 256 * 256, 3, device="cuda") * 0.5
    ws = torch.rand(T, 256 * 256, device="cuda")
    ms = timed(lambda: m.torso_composite_native(img, ws, lm, sc.bg_coords.cuda(), sc.bg_color.cuda(), want_maps=False), a.reps)
    lines.append({"what": "torso-SR field + composite alone (k_torso_sr)", "frames": T, "ms": ms, "ms_per_frame": ms / T})
    if T <= 16:   # the frame-by-frame host path is slow: only for small clips
        m.torso_backend, m.sr_net.backend = "torch", "torch"
        ms = timed(lambda: m.render_clip(poses, sc.intrinsics, 256, 256, **kw), max(1, a.reps // 2), warm=1)
        lines.append({"what": "torso-SR clip, host-side torso field + PyTorch SR (frame by frame)", "frames": T, "ms": ms, "fps": T / ms * 1e3})
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = measure(a.frames, a.reps)
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
