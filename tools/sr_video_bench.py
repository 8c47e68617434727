"""tools/sr_video_bench.py -- what the video frames of the SR checkpoints cost on one GPU: ms per frame of a clip from the driver's
batch to uint8 frames on the host, for RADNeRFwithSR and RADNeRFTorsowithSR (synthetic states at 256x256 -> 512x512).  Prints JSON
lines (device name and power limit first).

  SR head alone, on the same 256x256 frames:
    sr_f32_to_uint8_d2h   gfpp_sr_forward (fp32 planar [F,3,512,512]) + torch to_uint8 + copy to the host
    sr_u8_d2h             gfpp_sr_forward_video writing uint8 [F,512,512,3] only + copy to the host
  whole clip through driver.py:
    clip_f32_to_uint8_d2h render_driver_batch (fp32) -> video_uint8 -> .cpu()   (the driver's stacked path before the uint8 epilogue)
    clip_u8_d2h           render_driver_batch(as_uint8=True).cpu()             (stacked: the whole clip on the GPU, then one copy)
    clip_streamed         iter_video_frames: chunks double-buffered through pinned host memory while the next chunk renders

Arms alternate within each repetition (A B C, A B C, ...) after a warm-up of every arm; each timing is CUDA events around work that
ends on the host (the copy to the host synchronises).  The median over repetitions is reported.

    python tools/sr_video_bench.py [--frames 250] [--reps 5] [--out out/sr_video_bench.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import driver  # noqa: E402
from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.config import may_hparams  # noqa: E402
from genefaceplusplus_b200.dist import to_uint8  # noqa: E402


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


def alternate(arms, reps):
    """arms: {name: fn}.  One warm-up call of every arm, then `reps` rounds running the arms in turn; -> {name: [ms, ...]}."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(ms(fn))
    return times


def batch_for(T, torso):
    sc = scn.Scene(H=256, W=256, T=T, torso=torso, max_steps=16, density_scale=8.0)
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"].cuda() for f in fis], "rays_d": [f["rays_d"].cuda() for f in fis], "poses": [f["poses"].cuda() for f in fis],
            "cond_wins": [scn.cond_window(sc.cond, t, 3).cuda() for t in range(T)], "bg_coords": sc.bg_coords.cuda(),
            "bg_img": sc.bg_color.reshape(1, -1, 3).cuda(), "eye_area_percent": torch.full((T, 1), 0.37).cuda(),
            "lm68": scn.lm68_sequence(T).cuda()}


def model(which):
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR, RADNeRFwithSR
    hp = may_hparams(with_sr=True, add_eye_blink_cond=True, eye_blink_dim=4, smo_win_size=3, max_steps=16)
    if which == "head_sr":
        m = RADNeRFwithSR(hp)
        m.load_state_dict(scn.make_head_sr_state(hp), strict=True)
    else:
        hp["torso_head_aware"] = True
        m = RADNeRFTorsowithSR(hp)
        m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = 8.0
    return m.cuda().eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=250)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sr_video_bench needs a CUDA device (there is nothing to measure on the CPU)")
    T = a.frames
    lines = [{"what": "context", "frames": T, "reps": a.reps, **device_info()}]

    def report(which, times):
        for k, v in times.items():
            v = sorted(v)
            lines.append({"model": which, "arm": k, "ms_per_frame": v[len(v) // 2] / T, "min_ms_per_frame": v[0] / T,
                          "max_ms_per_frame": v[-1] / T})
            print(json.dumps(lines[-1]), flush=True)

    print(json.dumps(lines[0]), flush=True)
    for which in ("head_sr", "torso_sr"):
        m = model(which)
        batch = batch_for(T, which == "torso_sr")
        fpc = driver.SR_FRAMES_PER_CALL
        if which == "head_sr":   # the SR head alone, on the same input frame repeated
            rgb = (scn.hashed_uniform(256 * 256 * 3, 7, 0.5) + 0.5).cuda().view(1, -1, 3).expand(T, -1, -1).contiguous()
            u8 = torch.empty(T, 512, 512, 3, dtype=torch.uint8, device="cuda")
            f32 = torch.empty(T, 3, 512, 512, device="cuda")
            sr = m.sr_net
            report("sr_head", alternate({
                "sr_f32_to_uint8_d2h": lambda: to_uint8(sr.forward_native(rgb, noise_mode="const", clamp=True, out=f32,
                                                                          frames_per_call=fpc).permute(0, 2, 3, 1)).cpu(),
                "sr_u8_d2h": lambda: sr.forward_native(rgb, noise_mode="const", clamp=True, u8_out=u8, frames_per_call=fpc).cpu(),
            }, a.reps))
            del rgb, u8, f32

        def streamed():
            for c in driver.iter_video_frames(m, batch, frames_per_call=fpc, sr_noise_mode="const"):
                c.numpy()   # what a writer reads; the chunk is reused after the next advance

        report(which, alternate({
            "clip_f32_to_uint8_d2h": lambda: driver.video_uint8(driver.render_driver_batch(m, batch, sr_noise_mode="const")).cpu(),
            "clip_u8_d2h": lambda: driver.render_driver_batch(m, batch, as_uint8=True, sr_noise_mode="const").cpu(),
            "clip_streamed": streamed,
        }, a.reps))
        lines.append({"model": which, "peak_allocated_MiB": torch.cuda.max_memory_allocated() / 2 ** 20})
        print(json.dumps(lines[-1]), flush=True)
        del m, batch
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
