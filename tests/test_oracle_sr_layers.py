"""oracle/sr_emulate.py's float64 per-layer restatement of the SR kernels (`layer_f64`), pinned on the CPU.

Without its roundings (kernel=False: float64 fold of the weights, the module's 0.2 and sqrt 2) the chain of the four layers
must be the `Superresolution` module run in float64 -- to ~1e-12 relative, i.e. every layout convention of the restatement
(im2col tap order, the up-sampling layer's output phases, the closed-form skip up-sampling, the toRGB and skip sums) is the
module's.  tests/test_gpu_sr_layers.py then holds each kernel to this function on the kernel's own input."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.superres import Superresolution
from oracle.sr_emulate import layer_f64, rn16, ulp16

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _net():
    meta = json.loads(bytes(np.load(os.path.join(GOLD, "sr_head.npz"))["meta"]).decode())
    net = Superresolution(channels=3).eval()
    net.load_state_dict(scn.synthetic_sr_state({k: tuple(v) for k, v in meta["shapes"].items()}, seed=3), strict=False)
    return net


def _chain(fw, x, noise):
    """The four layers of layer_f64 without roundings: x [F,3,R,R] -> x0b, img0, img (NCHW like the module)."""
    rgb = x.permute(0, 2, 3, 1)
    x0a = layer_f64(fw, "in", rgb, noise[0], kernel=False)["v"]
    l0 = layer_f64(fw, 0, x0a, noise[1], skip=rgb, kernel=False)
    x1a = layer_f64(fw, 1, l0["v"], noise[2], kernel=False)["v"]
    img = layer_f64(fw, 2, x1a, noise[3], skip=l0["img"], kernel=False)["img"]
    return [t.permute(0, 3, 1, 2) for t in (l0["v"], l0["img"], img)]


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


def test_rn16_is_one_rounding_of_float64():
    """rn16 / ulp16 against numpy's direct float64 -> binary16 conversion, on normal and subnormal values and on exact ties
    (a tie of binary16 that float64 -> float32 -> float16 would break the other way is included)."""
    g = np.random.default_rng(7)
    v = np.concatenate([g.normal(0, 1, 20000) * 2.0 ** g.integers(-26, 8, 20000),
                        (np.arange(-3000, 3000) + 0.5) * 2.0 ** -24,               # ties in the subnormal range
                        (2048 + np.arange(0, 2048, 2) + 1.0) * 2.0 ** -12,       # ties between normal binary16 values
                        [1.0 + 2.0 ** -11 + 2.0 ** -40, 0.0, 256.0, -256.0, 2.0 ** -14, 2.0 ** -24]])
    got = rn16(torch.from_numpy(v)).numpy()
    assert np.array_equal(got, v.astype(np.float16).astype(np.float64))
    h = v.astype(np.float16)
    u = ulp16(torch.from_numpy(h.astype(np.float64))).numpy()
    assert np.array_equal(u, np.spacing(np.abs(h)).astype(np.float64))


def test_layer_chain_equals_the_module_in_float64():
    """256^2 with the 'const' noise planes: the rounding-free chain against Superresolution.double() (its blocks: forward()
    itself casts to fp32)."""
    net = _net()
    fw = net.folded_weights(torch.float64)
    netd = copy.deepcopy(net).double()
    x = scn.hashed_uniform(3 * 256 * 256, 78, 1.0).reshape(1, 3, 256, 256).double() + 0.5
    noise = [l.noise_const.double() * l.noise_strength.double() for l in netd._layers()]
    x0b, img0, img = _chain(fw, x, noise)
    w = torch.ones(netd.w_dim, dtype=torch.float64)
    with torch.no_grad():
        feat, ref0 = netd.block0(x, x, w, "const")
        _, ref = netd.block1(feat, ref0, w, "const")
    e = [_rel(x0b, feat), _rel(img0, ref0), _rel(img, ref)]
    print(f"256^2 const noise: relative max error x0b {e[0]:.2e}, img0 {e[1]:.2e}, image {e[2]:.2e}")
    assert max(e) <= 1e-12, e


@pytest.mark.parametrize("R", [128, 384])
def test_layer_chain_equals_the_blocks_at_other_sizes(R):
    """The sizes forward() does not take: block0 / block1 called directly, noise 'none'; at 128^2 two frames (the second the
    complement of the first).  Also: computing a subset of rows (how the GPU test covers 1024^2) gives those rows of the full
    result."""
    net = _net()
    fw = net.folded_weights(torch.float64)
    netd = copy.deepcopy(net).double()
    x = scn.hashed_uniform(3 * R * R, 11 + R, 1.0).reshape(1, 3, R, R).double() + 0.5
    if R == 128:
        x = torch.cat([x, 1.0 - x], 0)
    x0b, img0, img = _chain(fw, x, [None] * 4)
    w = torch.ones(netd.w_dim, dtype=torch.float64)
    with torch.no_grad():
        feat, ref0 = netd.block0(x, x, w, "none")
        _, ref = netd.block1(feat, ref0, w, "none")
    e = [_rel(x0b, feat), _rel(img0, ref0), _rel(img, ref)]
    print(f"{R}^2 no noise: relative max error x0b {e[0]:.2e}, img0 {e[1]:.2e}, image {e[2]:.2e}")
    assert img.shape == (x.shape[0], 3, 2 * R, 2 * R) and max(e) <= 1e-12, e
    rows = torch.tensor([0, 1, R // 2 + 3, R - 1])
    x0bh = x0b.permute(0, 2, 3, 1).half()
    full, part = layer_f64(fw, 1, x0bh), layer_f64(fw, 1, x0bh, rows=rows)
    out_rows = torch.stack([2 * rows, 2 * rows + 1], 1).reshape(-1)
    same = lambda a, b: torch.allclose(a, b, rtol=1e-13, atol=1e-13)   # noqa: E731  (GEMM blocking may differ with the row count)
    assert same(part["v"], full["v"][:, out_rows]) and same(part["S"], full["S"][:, out_rows])
    x1ah = full["v"].half()
    full2, part2 = layer_f64(fw, 2, x1ah, skip=img0.permute(0, 2, 3, 1)), layer_f64(fw, 2, x1ah, skip=img0.permute(0, 2, 3, 1), rows=out_rows)
    for k in ("v", "img", "rgbS", "dot", "skip"):
        assert same(part2[k], full2[k][:, out_rows]), k
