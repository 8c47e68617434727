"""tools/yuv_bench.py -- what planar I420 frames cost and save on one GPU, for a 250-frame clip of the 512x512 head + torso bench
scene (fp16, density_scale 8, T_thresh 0.01, random-init May weights) and of the torso-SR model (synthetic state, 256x256 NeRF ->
512x512 SR frames).  Prints JSON lines, the device name and power limit first.

    kernel        gfpp_rgb_u8_to_i420 alone on 512x512 frames: CUDA events around `--launches` back-to-back launches, per frame;
                  the 32-bit kernel (aligned buffers) and the byte kernel (output one byte off); bytes moved over kernel time
    clip          render_clip(as_uint8=True) against render_clip(as_yuv420=True), frames left on the device
    stream        driver.iter_video_frames, uint8 RGB against I420 chunks, ending with every frame in pinned host memory
    host          the CPU conversion the I420 frames take off the writer's path: video.i420_reference (numpy) per 512x512 frame,
                  and ffmpeg's own rgb24 -> yuv420p (rawvideo in, rawvideo out, timed against a yuv420p pass-through) only where an
                  ffmpeg binary exists

Arms alternate within every repetition after one warm-up call of each; GPU arms are timed with CUDA events around work that ends
in a synchronise (the streamed arms end on the host).  Medians over the repetitions, with min and max.  Before timing, the first
chunk of each I420 arm is checked byte for byte against video.i420_reference of the uint8 arm's frames.

    python tools/yuv_bench.py [--frames 250] [--reps 5] [--launches 50] [--out out/yuv_bench.jsonl]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import driver, video  # noqa: E402
from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.config import may_hparams  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR  # noqa: E402

S = 512                       # frame size of both models' video
HBM_TB_S = 3.35               # H100 SXM data sheet; a bound, not a measurement


def device_info():
    info = {"device": torch.cuda.get_device_name(0), "ffmpeg": shutil.which("ffmpeg")}
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


def alternate(arms, reps):
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(ms(fn))
    return times


def stats(v, per):
    v = sorted(x / per for x in v)
    return {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}


def kernel_lines(launches, reps):
    fb = video.i420_frame_bytes(S, S)
    out = []
    for F in (64, 250):
        rgb = torch.randint(0, 256, (F, S, S, 3), dtype=torch.uint8, device="cuda")
        big = torch.empty(F * fb + 4, dtype=torch.uint8, device="cuda")
        aligned, off = big[:F * fb], big[1:1 + F * fb]
        assert torch.equal(video.rgb_u8_to_i420(rgb, S, S, out=aligned).cpu()[:2].view(2, fb),
                           torch.from_numpy(video.i420_reference(rgb[:2].cpu().numpy())))

        def run(o):
            def fn():
                for _ in range(launches):
                    video.rgb_u8_to_i420(rgb, S, S, out=o)
            return fn

        t = alternate({"vector": run(aligned), "bytes": run(off)}, reps)
        moved = F * (S * S * 3 + fb)
        for k, v in t.items():
            st = stats(v, launches * F)
            out.append({"what": "kernel", "path": k, "frames_per_launch": F, "us_per_frame": 1e3 * st["median"],
                        "min_us_per_frame": 1e3 * st["min"], "max_us_per_frame": 1e3 * st["max"],
                        "GB_s": moved / (st["median"] * F * 1e-3) / 1e9, "share_of_datasheet_hbm": moved / (st["median"] * F * 1e-3) / (HBM_TB_S * 1e12)})
        del rgb, big
    return out


def host_lines(frames):
    rng = np.random.default_rng(0)
    rgb = rng.integers(0, 256, (frames, S, S, 3), dtype=np.uint8)
    video.i420_reference(rgb[:1])
    t0 = time.perf_counter()
    video.i420_reference(rgb)
    out = [{"what": "host", "conversion": "numpy i420_reference", "frames": frames, "ms_per_frame": 1e3 * (time.perf_counter() - t0) / frames}]
    ff = shutil.which("ffmpeg")
    if ff:
        raw = rgb.tobytes()
        yuv = video.i420_reference(rgb).tobytes()

        def run(pix, data):
            cmd = [ff, "-v", "error", "-f", "rawvideo", "-pix_fmt", pix, "-s", f"{S}x{S}", "-i", "-", "-f", "rawvideo", "-pix_fmt", "yuv420p", "-"]
            t = time.perf_counter()
            subprocess.run(cmd, input=data, capture_output=True, check=True)
            return time.perf_counter() - t

        run("rgb24", raw)
        conv = min(run("rgb24", raw) for _ in range(3))
        copy = min(run("yuv420p", yuv) for _ in range(3))
        out.append({"what": "host", "conversion": "ffmpeg rgb24 -> yuv420p minus yuv420p pass-through", "frames": frames,
                    "ms_per_frame": 1e3 * (conv - copy) / frames, "rgb24_ms_per_frame": 1e3 * conv / frames,
                    "yuv420p_ms_per_frame": 1e3 * copy / frames})
    else:
        out.append({"what": "host", "conversion": "ffmpeg", "measured": False, "reason": "no ffmpeg binary on PATH"})
    return out


def torso512(T):
    sc = scn.Scene(H=S, W=S, T=T, torso=True, density_scale=8.0)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m.mlp_precision = "fp16"
    m = m.cuda().eval()
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    kw = dict(cond_feat=m.cal_cond_feat_clip(sc.cond.cuda())[:T], pose6=scn.convert_poses(poses.cpu()).cuda(), bg_coords=sc.bg_coords.cuda(),
              bg_color=sc.bg_color.cuda(), T_thresh=sc.T_thresh, frames_per_call=64)
    clip = lambda **f: m.render_clip(poses, sc.intrinsics, S, S, **kw, **f)   # noqa: E731
    return m, sc, clip


def torso_sr(T):
    hp = may_hparams(with_sr=True, add_eye_blink_cond=True, eye_blink_dim=4, smo_win_size=3, max_steps=16, torso_head_aware=True)
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = 8.0
    m = m.cuda().eval()
    sc = scn.Scene(H=256, W=256, T=T, torso=True, max_steps=16, density_scale=8.0)
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    kw = dict(cond_seq=sc.cond.cuda(), eye_area_percent=torch.full((T,), 0.37), max_steps=16, T_thresh=sc.T_thresh,
              bg_color=sc.bg_color.cuda(), bg_coords=sc.bg_coords.cuda(), lm68_seq=scn.lm68_sequence(T).cuda(), sr_noise_mode="const")
    clip = lambda **f: m.render_clip(poses, sc.intrinsics, 256, 256, **kw, **f)   # noqa: E731
    return m, sc, clip


def batch_for(sc, m, T):
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"].cuda() for f in fis], "rays_d": [f["rays_d"].cuda() for f in fis], "poses": [f["poses"].cuda() for f in fis],
            "cond_wins": [scn.cond_window(sc.cond, t, m.smo_win_size).cuda() for t in range(T)], "bg_coords": sc.bg_coords.cuda(),
            "bg_img": sc.bg_color.reshape(1, -1, 3).cuda(), "eye_area_percent": torch.full((T, 1), 0.37).cuda(), "lm68": scn.lm68_sequence(T).cuda()}


def model_lines(which, T, reps):
    m, sc, clip = torso512(T) if which == "torso512" else torso_sr(T)
    fb = video.i420_frame_bytes(S, S)
    u8 = torch.empty((T, S * S, 3) if which == "torso512" else (T, S, S, 3), dtype=torch.uint8, device="cuda")
    yuv = torch.empty(T, fb, dtype=torch.uint8, device="cuda")
    parity = torch.equal(clip(as_yuv420=True, out=yuv)[:4].cpu(), torch.from_numpy(video.i420_reference(clip(as_uint8=True, out=u8)[:4].cpu().reshape(4, S, S, 3).numpy())))
    out = [{"what": "parity", "model": which, "i420_equals_reference_of_uint8": parity}]
    t = alternate({"u8": lambda: clip(as_uint8=True, out=u8), "yuv420": lambda: clip(as_yuv420=True, out=yuv)}, reps)
    for k, v in t.items():
        st = stats(v, T)
        out.append({"what": "clip", "model": which, "format": k, "frames": T, "ms_per_frame": st["median"], "min_ms_per_frame": st["min"],
                    "max_ms_per_frame": st["max"], "frames_per_s": 1e3 / st["median"]})
    del u8, yuv
    batch = batch_for(sc, m, T)
    fpc = 32 if which == "torso512" else driver.SR_FRAMES_PER_CALL

    def streamed(**f):
        def fn():
            for c in driver.iter_video_frames(m, batch, frames_per_call=fpc, T_thresh=sc.T_thresh, sr_noise_mode="const", **f):
                c.numpy()   # what a writer reads; the chunk is reused after the next advance
        return fn

    t = alternate({"u8": streamed(), "yuv420": streamed(as_yuv420=True)}, reps)
    for k, v in t.items():
        st = stats(v, T)
        out.append({"what": "stream", "model": which, "format": k, "frames": T, "frames_per_call": fpc, "host_bytes_per_frame": fb if k == "yuv420" else 3 * S * S,
                    "ms_per_frame": st["median"], "min_ms_per_frame": st["min"], "max_ms_per_frame": st["max"], "frames_per_s": 1e3 / st["median"]})
    del m, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=250)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("yuv_bench needs a CUDA device (there is nothing to measure on the CPU)")
    lines = [{"what": "context", "frames": a.frames, "reps": a.reps, "launches": a.launches, **device_info()}]
    print(json.dumps(lines[0]), flush=True)
    for part in (lambda: kernel_lines(a.launches, a.reps), lambda: model_lines("torso512", a.frames, a.reps),
                 lambda: model_lines("torso_sr", a.frames, a.reps), lambda: host_lines(min(a.frames, 50))):
        for ln in part():
            lines.append(ln)
            print(json.dumps(ln), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
