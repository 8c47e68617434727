"""tools/torso_sr_train_bench.py -- timings of the trainable torso-SR field (gfpp.h section I), one JSON line.

    python tools/torso_sr_train_bench.py [--iters 20] [--warmup 5]

CUDA events around each leg, median over --iters after --warmup, on the synthetic torso-SR state of the golden
(oracle/torso_sr_train.golden_state, head-aware, code dim 8), head-aware inputs at every point:
  * forward_torso in training mode, forward and forward + backward, at 65 536 (a 256 x 256 frame, the task's size) and 262 144 points
    (the fused libgfpp kernels);
  * the same in eager PyTorch, fp32 (F.linear over train_ops.grid_encode with input gradients; TF32 off) and under fp16 autocast.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from genefaceplusplus_b200 import train_ops  # noqa: E402
from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR  # noqa: E402
from oracle import torso_sr_train as tst  # noqa: E402
from torso_train_bench import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    hp = tst.golden_hparams("a")
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(tst.golden_state(hp), strict=False)
    m = m.cuda().train()
    P = tst.model_params(m)
    lm68 = tst.golden_lm68().cuda()
    idx = torch.tensor([1], device="cuda")
    out = {}

    def eager(x, c, img, ws):
        return tst.eager_torso_sr(m, P, x, lm68, c, img, ws, train_ops.grid_encode)

    def autocast(x, c, img, ws):
        with torch.autocast("cuda", dtype=torch.float16):
            return eager(x, c, img, ws)

    for M in (65536, 262144):
        pts = tst.golden_points(M, seed=M)
        x, img, ws = pts["x"].cuda(), pts["image"].cuda(), pts["weights_sum"].cuda()
        legs = {"fused": lambda x, c, img, ws: m.forward_torso(x, None, c, img, ws, lm68=lm68), "eager_fp32": eager,
                "eager_fp16_autocast": autocast}
        for name, f in legs.items():
            def fwd():
                with torch.no_grad():
                    f(x, m.torso_individual_codes[idx], img, ws)

            def fwd_bwd():
                m.zero_grad(set_to_none=True)
                a, c, d = f(x, m.torso_individual_codes[idx], img, ws)
                (a.float().sum() + c.float().sum() + d.float().sum()).backward()
            out[f"{name}.fwd_ms@{M}"] = timed(fwd, args.iters, args.warmup)
            out[f"{name}.fwd_bwd_ms@{M}"] = timed(fwd_bwd, args.iters, args.warmup)
    name, power = card()
    print(json.dumps({"tool": "torso_sr_train_bench", "gpu": name, "power_limit": power, "iters": args.iters, "warmup": args.warmup, **out}))


if __name__ == "__main__":
    main()
