"""The torch path's autograd of Superresolution against the reference's own module (tests/golden/sr_head_grad.npz, written by
oracle/make_sr_grad_golden.py from radnerf_sr.py:15-48 on CPU with autograd).

This pins the backward's semantics to the reference, in the plain state and in a loud one where the +256 clamp and the leaky
branch are live: the slope of the leaky ReLU, the zero past the clamp, the toRGB clamp, the adjoint of the up-sampled skip and
the noise strengths' sum of gradient times noise_const.  Both sides run in fp32 with different summation orders, so the bar is
fp32 rounding over the sums involved: each sampled element within 1e-4 of the tensor's largest sampled magnitude (the absolute
sum / numel for the scale when the sample is all zero), sum within 1e-4 of the absolute sum, norm within 1e-4 relative.
tests/test_gpu_sr_grad.py then holds the native backward to this path."""
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.superres import Superresolution

GOLD = os.path.join(os.path.dirname(__file__), "golden", "sr_head_grad.npz")
TOL = 1e-4


def _loud(st):
    st = dict(st)
    for name in ("block0.conv0", "block0.conv1", "block1.conv0", "block1.conv1"):
        b, w = st[name + ".bias"].clone(), st[name + ".weight"].clone()
        b[0::4], b[1::4], b[2::4] = 320.0, -60.0, 0.0
        w[2::4] *= 1e-10
        st[name + ".bias"], st[name + ".weight"] = b, w
    return st


@pytest.mark.parametrize("tag", ["plain", "loud"])
def test_torch_path_gradients_match_the_reference(tag):
    gold = np.load(GOLD)
    net = Superresolution(channels=3)
    net.backend = "torch"
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    st = scn.synthetic_sr_state(shapes, seed=3)
    net.load_state_dict(_loud(st) if tag == "loud" else st, strict=False)
    x = (scn.hashed_uniform(3 * 256 * 256, 78, 1.0).reshape(1, 3, 256, 256) + 0.5).requires_grad_(True)
    G = scn.hashed_uniform(3 * 512 * 512, 91, 1.0).reshape(1, 3, 512, 512) / (3 * 512 * 512)
    (net(x, noise_mode="const") * G).sum().backward()
    pairs = [("input", x.grad)] + [(n, p.grad) for n, p in net.named_parameters()]
    assert len(pairs) == 29
    for name, g in pairs:
        key = f"{tag}/{name}"
        g = g.double().reshape(-1)
        idx, val, stats = gold[key + "/idx"], gold[key + "/val"], gold[key + "/stats"]
        got = g[torch.from_numpy(idx)].numpy()
        scale = max(np.abs(val).max(), stats[1] / g.numel(), 1e-30)
        assert np.abs(got - val).max() <= TOL * scale, (name, np.abs(got - val).max() / scale)
        assert abs(float(g.sum()) - stats[0]) <= TOL * stats[1] + 1e-30, name
        assert abs(float(g.norm()) - stats[2]) <= TOL * stats[2] + 1e-30, name
