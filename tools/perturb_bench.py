"""Time one 512x512 head+torso render() with perturb=True against perturb=False (the reference's validation call vs its inference call).

    python tools/perturb_bench.py [--reps 21] [--warmup 5] [--precision fp32]

Both legs run RADNeRFTorso.render in eval mode on the bench scene (density_scale 8, max_steps 16, T_thresh 0.01), interleaved, each
timed with CUDA events around the whole call (conditioning nets, the torch.rand(N) draw of perturb=True, libgfpp's render and the
result views).  The jitter moves where each ray starts marching, so the sample count S differs slightly between the legs; both S
values are reported.  Prints one JSON line with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRFTorso  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "fp16", "bf16x3", "bf16", "robust"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perturb_bench needs a GPU")
    sc = scn.Scene(H=args.size, W=args.size, T=2, torso=True, density_scale=8.0)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m.mlp_precision = args.precision
    m = m.cuda().eval()
    fi = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in sc.frame_inputs(0).items()}

    def call(perturb):
        return m.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=0, staged=False, bg_color=fi["bg_color"],
                        perturb=perturb, force_all_rays=False, T_thresh=sc.T_thresh, **sc.hparams)

    torch.cuda.manual_seed(0)
    for _ in range(args.warmup):
        call(False); call(True)
    times = {False: [], True: []}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(args.reps):
        for p in (False, True):
            ev[0].record()
            call(p)
            ev[1].record()
            ev[1].synchronize()
            times[p].append(ev[0].elapsed_time(ev[1]))
    # the sample counts of both legs, from the same frame (noise: the draw render(perturb=True) makes after this seed)
    N = args.size * args.size
    cf = m.cal_cond_feat(fi["cond"]).view(1, -1)
    torch.cuda.manual_seed(0)
    noise = torch.rand(N, device="cuda")
    S = {}
    for p in (False, True):
        res = m.render_frames(cf, rays_o=fi["rays_o"].view(1, -1, 3), rays_d=fi["rays_d"].view(1, -1, 3), pose6=fi["poses"], bg_coords=fi["bg_coords"],
                              bg_color=fi["bg_color"], dt_gamma=sc.hparams["dt_gamma"], max_steps=sc.hparams["max_steps"], T_thresh=sc.T_thresh,
                              want_stats=True, noise=noise if p else None)
        S[p] = int(res["stats"][0, 2])
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        power = f"unavailable ({e})"
    med = {p: statistics.median(t) for p, t in times.items()}
    out = {"tool": "perturb_bench", "gpu": torch.cuda.get_device_name(0), "power_limit": power, "size": args.size, "precision": args.precision,
           "reps": args.reps, "ms_perturb_false": med[False], "ms_perturb_true": med[True],
           "ms_spread_false": [min(times[False]), max(times[False])], "ms_spread_true": [min(times[True]), max(times[True])],
           "overhead_pct": 100.0 * (med[True] / med[False] - 1.0), "S_perturb_false": S[False], "S_perturb_true": S[True]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
