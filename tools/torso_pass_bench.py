"""tools/torso_pass_bench.py -- the torso part of the torso training steps, composed (README recipe) against torso_pass() (gfpp.h
section M), one JSON line.

    python tools/torso_pass_bench.py [--rounds 7] [--iters 10] [--warmup 3]

For both torso models, at 65 536 and 262 144 rays of a scene.Scene torso frame (256 x 256 and 512 x 512), with the frozen head in
fp32 and in fp16 (under autocast, as the torso configs' amp: true runs it):
  * torso: the torso part alone -- mask, field forward, composite, the task loss and its backward -- on a fixed frozen_head output;
  * step: frozen_head + the torso part.
CUDA events around each leg, the composed and fused legs alternating within each round; per leg the median over rounds of the
median of --iters after --warmup.  The card's name and power limit are read in the same run.
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
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR  # noqa: E402
from oracle import torso_sr_train as tst  # noqa: E402
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
    return ts[len(ts) // 2]


def composite(mask, alpha, color, image, ws, bg):
    N = mask.shape[0]
    ta = torch.zeros(N, 1, device="cuda")
    tc = torch.zeros(N, 3, device="cuda")
    ta[mask] = alpha
    tc[mask] = color
    trgb = tc * ta + bg.reshape(-1, 3) * (1 - ta)
    return {"torso_alpha_map": ta, "torso_rgb_map": trgb, "rgb_map": (image + (1 - ws).unsqueeze(-1) * trgb).clamp(0, 1)}


def composed(m, sr, image, ws, bgc, pose6, code, bg, lm68):
    if sr:
        G = m.grid_size
        occ = F.grid_sample(m.density_grid_torso.view(1, 1, G, G), bgc.view(1, -1, 1, 2), align_corners=True).view(-1)
        mask = occ > min(m.density_thresh_torso, m.mean_density_torso)
        a, c, d = m.forward_torso(bgc[mask], None, code, image[mask], ws[mask].unsqueeze(-1), lm68=lm68)
    else:
        mask = m.torso_mask(bgc)
        a, c, d = m.forward_torso(bgc[mask], pose6, code)
    res = composite(mask, a, c, image, ws, bg)
    res["deform"] = d
    return res


def loss_of(res, gt, sr):
    a = res["torso_alpha_map"].clamp(1e-5, 1 - 1e-5)
    loss = ((res["torso_rgb_map"] - gt) ** 2).mean() + 1e-4 * (-a * torch.log2(a) - (1 - a) * torch.log2(1 - a)).mean()
    return loss + 1e-3 * res["deform"].abs().mean() if sr else loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = card()
    out = {"card": name, "power_limit": power, "unit": "ms, median"}
    for side in (256, 512):
        sc = scn.Scene(H=side, W=side, T=4, torso=True, density_scale=tt.GOLDEN_DS)
        fi = sc.frame_inputs(1)
        ro, rd = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
        bgc, bg = fi["bg_coords"].cuda().reshape(-1, 2), fi["bg_color"].cuda()
        N = ro.shape[0]
        gt = tt.golden_target(N).cuda()
        pose6, lm68 = fi["poses"].cuda(), tst.golden_lm68().cuda()
        idx = torch.tensor([1], device="cuda")
        for cls in ("torso", "sr"):
            if cls == "torso":
                m = RADNeRFTorso(sc.hparams)
                m.load_state_dict(sc.state, strict=True)
                cond, kw = fi["cond"].cuda(), {}
            else:
                hp = tst.golden_hparams("b")
                m = RADNeRFTorsowithSR(hp)
                m.load_state_dict(tst.golden_state(hp), strict=False)
                m.density_bitfield.copy_(sc.state["density_bitfield"])
                cond, kw = scn.cond_window(sc.cond, 1, hp["smo_win_size"]), {"eye_area_percent": torch.tensor([0.3])}
                kw = {k: v.cuda() for k, v in kw.items()}
            m.density_scale = tt.GOLDEN_DS
            m = m.cuda().train()
            sr = cls == "sr"
            for prec in ("fp32", "fp16"):
                m.mlp_precision = prec
                amp = torch.autocast("cuda", dtype=torch.float16, enabled=prec == "fp16")
                with torch.no_grad(), amp:
                    feat = m.cal_cond_feat(cond.cuda(), **kw)

                def head():
                    with amp:
                        return m.frozen_head(ro, rd, feat, m.individual_embeddings[idx], max_steps=16)

                ws0, img0 = head()

                def torso(fused, ws, img):
                    m.zero_grad(set_to_none=True)
                    code = m.torso_individual_codes[idx]
                    with amp:
                        res = (m.torso_pass(img, ws, bgc, pose6, code, bg_color=bg, lm68=lm68) if fused else
                               composed(m, sr, img, ws, bgc, pose6, code, bg, lm68))
                        loss = loss_of(res, gt, sr)
                    loss.backward()

                legs = {"torso_composed": lambda: torso(False, ws0, img0), "torso_fused": lambda: torso(True, ws0, img0),
                        "step_composed": lambda: torso(False, *head()), "step_fused": lambda: torso(True, *head())}
                per = {k: [] for k in legs}
                for _ in range(args.rounds):
                    for k, fn in legs.items():
                        per[k].append(timed(fn, args.iters, args.warmup))
                key = f"{cls}_{N}_{prec}"
                out[key] = {k: round(sorted(v)[len(v) // 2], 4) for k, v in per.items()}
                out[key]["masked_pixels"] = int(m.torso_pass(img0, ws0, bgc, pose6, m.torso_individual_codes[idx], bg_color=bg,
                                                             lm68=lm68)["deform"].shape[0])
                print(key, out[key], file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
