"""oracle/make_sr_grad_golden.py -- golden gradients of the super-resolution head.

Runs only where /root/reference exists.  Builds the reference's `Superresolution(channels=3)` (radnerf_sr.py:15-48) on CPU through
oracle/ref_shim.py, as oracle/make_sr_golden.py does for its forward (the eg3ds ops take their pure-torch `_ref` paths on CPU), and
runs it with autograd and `noise_mode='const'` on the 256x256 input of sr_head.npz, for two states:
  * "plain": genefaceplusplus_b200.scene.synthetic_sr_state(shapes, seed=3), the state of tests/golden/sr_head.npz;
  * "loud":  the same with, per 3x3 layer, a quarter of the channels biased to +320 (past the +256 clamp), a quarter to -60
             (the leaky branch) and a quarter with weights x 1e-10 and no bias -- the variant of tests/test_gpu_sr_layers.py.
The loss is sum(out * G) with the closed-form upstream gradient G = hashed_uniform(seed 91) / (3 * 512 * 512), the size a
mean-reduced MSE gives, so nothing large is stored.  Per tensor (the input, then every parameter by name) the file keeps a fixed
subset of the gradient (every element of tensors up to 64 values, else 64 at hashed positions) and its sum, absolute sum and
L2 norm, in float64.

Usage:  python -m oracle.make_sr_grad_golden
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from oracle import ops, ref_shim  # noqa: E402

N_SUBSET = 64


def loud_state(st):
    st = dict(st)
    for name in ("block0.conv0", "block0.conv1", "block1.conv0", "block1.conv1"):
        b, w = st[name + ".bias"].clone(), st[name + ".weight"].clone()
        b[0::4], b[1::4], b[2::4] = 320.0, -60.0, 0.0
        w[2::4] *= 1e-10
        st[name + ".bias"], st[name + ".weight"] = b, w
    return st


def sr_input():
    return scn.hashed_uniform(3 * 256 * 256, 78, 1.0).reshape(1, 3, 256, 256) + 0.5


def upstream():
    return scn.hashed_uniform(3 * 512 * 512, 91, 1.0).reshape(1, 3, 512, 512) / (3 * 512 * 512)


def subset(n):
    """Fixed flat positions: all of a small tensor, else N_SUBSET hashed ones (the first and the last included)."""
    if n <= N_SUBSET:
        return np.arange(n)
    h = (np.arange(N_SUBSET - 2, dtype=np.uint64) * np.uint64(2654435761) + np.uint64(97)) % np.uint64(n)
    return np.unique(np.concatenate([[0, n - 1], h.astype(np.int64)]))


def main():
    cwd = os.getcwd()
    ops.build()
    ref_shim.install(ops)
    from modules.radnerfs.radnerf_sr import Superresolution
    with torch.no_grad():
        net = Superresolution(channels=3).eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    # block0 receives the same tensor as x and as the rgb skip and adds its toRGB output to the skip in place
    # (superresolution.py:251).  On CUDA its fp16 cast of x makes x a separate tensor; on CPU (no fp16) x aliases the skip
    # and autograd refuses the in-place add.  A copy of the skip restores the CUDA aliasing, with the same values.
    fwd0 = net.block0.forward
    net.block0.forward = lambda x, img, ws, **kw: fwd0(x, img.clone(), ws, **kw)
    out = {}
    for tag in ("plain", "loud"):
        st = scn.synthetic_sr_state(shapes, seed=3)
        net.load_state_dict(loud_state(st) if tag == "loud" else st, strict=False)
        net.zero_grad(set_to_none=True)
        x = sr_input().clone().requires_grad_(True)
        y = net(x.clone(), noise_mode="const")   # a copy, as the tasks pass it (radnerf_torso_sr.py:236)
        assert y.shape == (1, 3, 512, 512)
        (y * upstream()).sum().backward()
        for name, g in [("input", x.grad)] + [(n, p.grad) for n, p in net.named_parameters()]:
            assert g is not None, name
            g = g.detach().double().reshape(-1)
            idx = subset(g.numel())
            key = f"{tag}/{name}"
            out[key + "/idx"] = idx
            out[key + "/val"] = g[torch.from_numpy(idx)].numpy()
            out[key + "/stats"] = np.array([float(g.sum()), float(g.abs().sum()), float(g.norm())])
        print(tag, "out range", float(y.min()), float(y.max()))
    meta = dict(source="reference Superresolution (radnerf_sr.py:15-48) on CPU via oracle/ref_shim.py, autograd, noise_mode='const'",
                state="genefaceplusplus_b200.scene.synthetic_sr_state(shapes, seed=3); 'loud' per oracle/make_sr_grad_golden.loud_state",
                loss="sum(out * hashed_uniform(3*512*512, 91, 1.0) / (3*512*512))", torch=torch.__version__)
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    os.chdir(cwd)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "sr_head_grad.npz"), **out)
    print("wrote tests/golden/sr_head_grad.npz")


if __name__ == "__main__":
    main()
