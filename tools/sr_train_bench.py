"""Forward + backward time of the SR head per 256^2 frame: the native path (train_ops.sr_head, TF32 wgmma backward) against
autograd of the torch path (cuDNN), CUDA events after warm-up, with the card's name and power limit.

    python tools/sr_train_bench.py [--frames 1] [--iters 20]

Share of the TF32 peak is computed from algorithmic FLOPs counted from the shapes below (forward ~78 GFLOP per frame, backward
~155 GFLOP: dgrad and wgrad of the three GEMM layers, each as many FLOPs as the forward GEMM) over the measured time."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.superres import Superresolution

TF32_PEAK = 495e12   # H100 SXM dense TF32, data sheet, 700 W


def flops(R=256):
    px, px2 = R * R, 4 * R * R
    fwd = 2 * (px * 128 * 27 + px * 128 * 1152 + px * 256 * 1152 + px2 * 64 * 576 + px * 3 * 128 + px2 * 3 * 64)
    gemm = 2 * (px * 128 * 1152 + px * 256 * 1152 + px2 * 64 * 576)
    bwd = 2 * gemm + 2 * 2 * px * 128 * 27
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sr_train_bench needs a CUDA device")
    shapes = {k: tuple(v.shape) for k, v in Superresolution(channels=3).state_dict().items()}
    net = Superresolution(channels=3)
    net.load_state_dict(scn.synthetic_sr_state(shapes, seed=3), strict=False)
    net = net.cuda()
    x = (torch.rand(a.frames, 3, 256, 256, device="cuda")).requires_grad_(True)
    G = torch.randn(a.frames, 3, 512, 512, device="cuda") / (a.frames * 3 * 512 * 512)
    res = {}
    for backend in ("native", "torch"):
        net.backend = backend

        def step():
            net.zero_grad(set_to_none=True)
            x.grad = None
            (net(x, noise_mode="const") * G).sum().backward()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            step()
        e1.record()
        torch.cuda.synchronize()
        res[backend] = e0.elapsed_time(e1) / a.iters / a.frames
    fwd, bwd = flops()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"card": q, "frames": a.frames, "ms_per_frame_native": round(res["native"], 3), "ms_per_frame_torch": round(res["torch"], 3),
           "gflop_fwd_per_frame": round(fwd / 1e9, 1), "gflop_bwd_per_frame": round(bwd / 1e9, 1),
           "tf32_peak_share_native": round((fwd + bwd) / (res["native"] * 1e-3) / TF32_PEAK, 3),
           "note": "whole step (host fold, packing checks, forward, backward) over the TF32 data-sheet peak; not a kernel's share"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
