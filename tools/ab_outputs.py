#!/usr/bin/env python
"""Outputs of this tree against another checkout of the project on the bench workload's first 50-frame call (512x512 head+torso,
density_scale 8, max_steps 16, T_thresh 0.01), fp16 and robust:

  * weights_sum, depth and the per-frame stats (B_total, n_survivors, S, P): equal or not;
  * RGB max|delta| between the two trees;
  * RGB of both trees against the fp32 CPU oracle on frames 0 / 25 / 49, on the rays the kernel generates.

    python tools/ab_outputs.py --base DIR [--frames 50] [--oracle-frames 0,25,49]

Each tree renders in a subprocess of its own (both builds are named libgfpp); the frames go through a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRECISIONS = ("fp16", "robust")


def render(tree, out_dir, frames, oracle_frames):
    """In `tree`'s package: one render_frames call of `frames` frames per precision -> out_dir/<precision>.pt (with the generated
    rays of `oracle_frames`)"""
    sys.path.insert(0, tree)
    import torch
    from genefaceplusplus_b200 import scene as scn
    from genefaceplusplus_b200.renderer import RADNeRFTorso
    sc = scn.Scene(H=512, W=512, T=frames, torso=True, density_scale=8.0)
    poses = torch.stack([sc.pose(t) for t in range(frames)]).cuda()
    for prec in PRECISIONS:
        m = RADNeRFTorso(sc.hparams)
        m.load_state_dict(sc.state, strict=True)
        m.density_scale, m.mlp_precision = sc.density_scale, prec
        m = m.cuda().eval()
        feat = m.cal_cond_feat_clip(sc.cond.cuda())[:frames]
        with torch.no_grad():
            res = m.render_frames(feat, poses_c2w=poses, intrinsics=sc.intrinsics, H=512, W=512, pose6=scn.convert_poses(poses.cpu()).cuda(),
                                  bg_coords=sc.bg_coords.cuda(), bg_color=sc.bg_color.cuda(), dt_gamma=sc.hparams["dt_gamma"],
                                  max_steps=sc.hparams["max_steps"], T_thresh=sc.T_thresh, want_torso_maps=False, want_stats=True)
            rays = m.generate_rays(poses[oracle_frames], sc.intrinsics, 512, 512)
        torch.cuda.synchronize()
        torch.save({k: res[k].cpu() for k in ("rgb_map", "weights_sum", "depth_map", "stats")} | {"rays": tuple(r.cpu() for r in rays)},
                   os.path.join(out_dir, f"{prec}.pt"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="the other checkout (built)")
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--oracle-frames", default="0,25,49")
    ap.add_argument("--render", nargs=2, metavar=("TREE", "OUT"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    oracle_frames = [int(x) for x in args.oracle_frames.split(",")]
    if args.render:
        render(args.render[0], args.render[1], args.frames, oracle_frames)
        return
    import torch
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from genefaceplusplus_b200 import scene as scn
    from helpers import parity_report
    from oracle import ops
    from oracle.render import OracleModel
    ops.build()
    with tempfile.TemporaryDirectory() as tmp:
        dirs = {}
        for name, tree in (("base", os.path.abspath(args.base)), ("this", ROOT)):
            dirs[name] = os.path.join(tmp, name)
            os.makedirs(dirs[name])
            subprocess.run([sys.executable, os.path.abspath(__file__), "--base", args.base, "--frames", str(args.frames),
                            "--oracle-frames", args.oracle_frames, "--render", tree, dirs[name]], check=True)
        sc = scn.Scene(H=512, W=512, T=args.frames, torso=True, density_scale=8.0)
        orc = OracleModel(sc.state, sc.hparams)
        orc.density_scale = sc.density_scale
        report = {}
        for prec in PRECISIONS:
            b, t = (torch.load(os.path.join(dirs[n], f"{prec}.pt")) for n in ("base", "this"))
            r = {k: bool(torch.equal(b[k], t[k])) for k in ("weights_sum", "depth_map", "stats")}
            r["rays_equal"] = all(torch.equal(x, y) for x, y in zip(b["rays"], t["rays"]))
            r["rgb_max_abs_vs_base"] = (b["rgb_map"] - t["rgb_map"]).abs().max().item()
            r["oracle"] = {}
            for i, f in enumerate(oracle_frames):
                fi = sc.frame_inputs(f)
                ref = orc.render(t["rays"][0][i].view(1, -1, 3), t["rays"][1][i].view(1, -1, 3), fi["cond"], fi["bg_coords"], fi["poses"],
                                 bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **sc.hparams)
                r["oracle"][f] = {n: parity_report(x["rgb_map"][f], ref["rgb_map"].view(-1, 3), ref["knife"])["max_abs"] for n, x in (("base", b), ("this", t))}
            report[prec] = r
            print(f"{prec}: {json.dumps(r)}", flush=True)


if __name__ == "__main__":
    main()
