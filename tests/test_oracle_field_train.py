"""The training field's CPU checker (oracle/field_train.py): its autograd gradients against central finite differences of the same
function with float64 dense layers, at a few entries of every parameter downstream of the ambient grid (sigma and colour nets, the
ambient table).  Upstream of it (ambient net, position table) a perturbation moves the ambient coordinates across the grid's cells,
where the piecewise-linear interpolation has kinks, and the fp32 lookups quantise the coordinates: finite differences do not
converge there, and those gradients are checked against libgfpp and the training render instead (tests/test_gpu_field_train.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import scene as scn
from oracle import field_train as ft
from oracle import ops


@pytest.fixture(scope="module")
def case():
    ops.build()
    sc = scn.Scene(H=8, W=8, T=2, torso=False)
    g = torch.Generator().manual_seed(11)
    M = 200
    x = (torch.rand(M, 3, generator=g) - 0.5) * torch.tensor([1.6, 0.8, 1.6])
    d = F.normalize(torch.randn(M, 3, generator=g), dim=-1).double()
    cond = torch.randn(1, 64, generator=g, dtype=torch.float64) * 0.3
    code = sc.state["individual_embeddings"][1].double()
    w = [torch.randn(M, generator=g, dtype=torch.float64), torch.randn(M, 3, generator=g, dtype=torch.float64),
         torch.randn(M, 3, generator=g, dtype=torch.float64)]
    return sc, x, d, cond, code, w


def _loss(p, sc, x, d, cond, code, w):
    s, c, a = ft.field_forward(p, sc.hparams, x, d, cond, code)
    return (s * w[0]).sum() + (c * w[1]).sum() + (a * w[2]).sum()


def test_gradients_match_finite_differences(case):
    sc, x, d, cond, code, w = case
    p = ft.field_params(sc.state, torch.float64)
    _loss(p, sc, x, d, cond, code, w).backward()
    rng = np.random.default_rng(0)
    checked = 0
    keys = [k for k in ft.TRAINABLE if k.startswith(("sigma_net", "color_net", "ambient_embedder"))]
    for k in keys:
        grad = p[k].grad
        # the entries with the largest gradients (well above the fp32 grid lookups' rounding) plus one random one
        flat = grad.reshape(-1)
        idx = list(torch.topk(flat.abs(), 2).indices.tolist()) + [int(rng.integers(flat.numel()))]
        h = 1e-3 if k.endswith("embeddings") else 1e-5   # the table steps through the fp32 lookups: a larger step
        for i in idx:
            q = {kk: (vv.detach().clone() if torch.is_tensor(vv) else vv) for kk, vv in p.items()}
            q[k].reshape(-1)[i] += h
            lp = _loss(q, sc, x, d, cond, code, w).item()
            q[k].reshape(-1)[i] -= 2 * h
            lm = _loss(q, sc, x, d, cond, code, w).item()
            fd = (lp - lm) / (2 * h)
            scale = max(flat.abs().max().item(), 1e-12)
            tol = 5e-3 if k.endswith("embeddings") else 1e-4   # fp32 lookup rounding over ReLU kinks: measured 3e-3 at most
            assert abs(fd - flat[i].item()) <= tol * scale, (k, i, fd, flat[i].item())
            checked += 1
    assert checked == 3 * len(keys) == 18


def test_oracle_training_render_against_reference_golden():
    """oracle/field_train.render_train + backward against tests/golden/train_head.npz, the reference's own RADNeRF.render in training
    mode and its backward on the same inputs (oracle/make_train_golden.py measured 0 difference when it wrote the golden)."""
    import os
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_head.npz"))
    ops.build()
    sc = scn.Scene(H=32, W=32, T=4, torso=False, density_scale=8.0)
    p = ft.field_params(sc.state)
    emb = sc.state["individual_embeddings"].clone().requires_grad_(True)
    t = lambda k: torch.from_numpy(G[k])   # noqa: E731
    res = ft.render_train(p, sc.hparams, sc.state, t("rays_o"), t("rays_d"), t("cond_feat"), emb[2], t("bg_color"), 8.0, 16)
    ((res["rgb_map"].reshape(-1, 3) * t("coef_rgb")).sum() + (res["weights_sum"] * t("coef_ws")).sum() + (res["ambient"] * t("coef_amb")).sum()).backward()
    assert torch.equal(res["position"], t("position"))
    got = {k: res[k].detach() for k in ("rgb_map", "weights_sum", "ambient", "depth_map")}
    got.update({"grad." + k: p[k].grad for k in ft.TRAINABLE[:8]})
    got["grad.individual_code"] = emb.grad[2]
    for k, v in got.items():
        ref = t(k)
        e = (v.reshape(ref.shape) - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)
        assert e <= 1e-6, (k, e)
    for tname in ("position_embedder", "ambient_embedder"):
        gr = p[f"{tname}.embeddings"].grad
        ref = t(f"{tname}.sample_grad")
        assert (gr[t(f"{tname}.sample_idx")] - ref).abs().max().item() <= 1e-6 * ref.abs().max().item(), tname
