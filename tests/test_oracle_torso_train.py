"""The CPU checker of the trainable torso field (oracle/torso_train.py) against tests/golden/train_torso.npz, which holds the
reference's own RADNeRFTorso.forward_torso + backward (part a) and its torso training step (part b), and against finite differences
in float64."""
import os

import numpy as np
import pytest
import torch

from oracle import field_train as ft
from oracle import ops
from oracle import torso_train as tt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_torso.npz")
REL = 1e-6       # the checker runs the reference's arithmetic: 0 when the golden was made


@pytest.fixture(scope="module")
def case():
    ops.build()
    return tt.golden_scene(), np.load(GOLDEN)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def test_golden_a_forward_torso_and_backward(case):
    sc, z = case
    x = torch.from_numpy(z["a.x"])
    ca, cc, cd = (torch.from_numpy(z[k]) for k in ("a.coef_alpha", "a.coef_color", "a.coef_deform"))
    p = tt.torso_params(sc.state)
    codes = sc.state["torso_individual_codes"].clone().requires_grad_(True)
    trace = {}
    a, c, dx = tt.torso_forward(p, sc.hparams, x, torch.from_numpy(z["pose6"]), codes[torch.tensor([tt.GOLDEN_INDEX])], trace)
    ((a * ca).sum() + (c * cc).sum() + (dx * cd).sum()).backward()
    assert int((trace["x_pre_clamp"].abs() > 1).any(-1).sum()) > 0, "the golden must exercise the clamp"
    for k, o in (("alpha", a), ("color", c), ("deform", dx)):
        assert _rel(o.detach(), z[f"a.{k}"]) <= REL, k
    for k in tt.TRAINABLE[:6]:
        assert _rel(p[k].grad, z[f"a.grad.{k}"]) <= REL, k
    assert _rel(codes.grad[tt.GOLDEN_INDEX], z["a.grad.code"]) <= REL
    idx = torch.from_numpy(z["table_sample_idx"])
    assert _rel(p["torso_embedder.embeddings"].grad[idx], z["a.grad.table_sample"]) <= REL
    rows = torch.nonzero(codes.grad.abs().sum(-1)).reshape(-1).tolist()
    assert rows == [tt.GOLDEN_INDEX]


def test_golden_b_torso_training_step(case):
    sc, z = case
    index = torch.tensor([tt.GOLDEN_INDEX])
    hpar = ft.field_params(sc.state)
    p = tt.torso_params(sc.state)
    codes = sc.state["torso_individual_codes"].clone().requires_grad_(True)
    t = {k: torch.from_numpy(z[f"b.{k}"]) for k in ("rays_o", "rays_d", "bg_coords", "bg_color", "gt", "cond_feat")}
    res = tt.train_step(hpar, p, sc.hparams, sc.state, t["rays_o"], t["rays_d"], t["cond_feat"], sc.state["individual_embeddings"][index],
                        t["bg_coords"], torch.from_numpy(z["pose6"]), codes[index], t["bg_color"], tt.GOLDEN_DS, tt.GOLDEN_MAX_STEPS)
    tt.task_loss(res, t["gt"], tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    M, N = int(res["mask"].sum()), res["mask"].numel()
    assert 0 < M < N, "the mask must keep some pixels but not all"
    for k in ("torso_alpha_map", "torso_rgb_map", "rgb_map", "weights_sum"):
        assert _rel(res[k].detach().reshape(-1), z[f"b.{k}"].reshape(-1)) <= REL, k
    for k in tt.TRAINABLE[:6]:
        assert _rel(p[k].grad, z[f"b.grad.{k}"]) <= REL, k
    assert _rel(codes.grad[tt.GOLDEN_INDEX], z["b.grad.code"]) <= REL


def test_float64_gradients_match_finite_differences(case):
    """The float64 checker (what the GPU gradients are measured against) against central differences, at points away from ties."""
    sc, _ = case
    g = torch.Generator().manual_seed(3)
    x = torch.rand(64, 2, generator=g) * 2 - 1
    w = torch.randn(64, 6, generator=g, dtype=torch.float64)
    pose6 = sc.frame_inputs(tt.GOLDEN_FRAME)["poses"]
    trace = {}
    p = tt.torso_params(sc.state, torch.float64)
    tt.torso_forward(p, sc.hparams, x, pose6, sc.state["torso_individual_codes"][1].double(), trace)
    x = x[~tt.tie_mask(trace, 1e-4)]
    w = w[: x.shape[0]]

    def loss(pp):
        a, c, dx = tt.torso_forward(pp, sc.hparams, x, pose6, sc.state["torso_individual_codes"][1].double())
        return (torch.cat([a, c, dx], -1) * w).sum()

    p = tt.torso_params(sc.state, torch.float64)
    loss(p).backward()
    # the canonical net only: the deform net reaches the grid through its fp32 input, as in the reference
    for k in ("torso_canonicial_net.net.0.weight", "torso_canonicial_net.net.1.weight", "torso_canonicial_net.net.2.weight"):
        W = p[k]
        for (i, j) in ((0, 0), (1, 3), (W.shape[0] - 1, W.shape[1] - 1)):
            h = 1e-6
            with torch.no_grad():
                W[i, j] += h
                lp = loss(p).item()
                W[i, j] -= 2 * h
                lm = loss(p).item()
                W[i, j] += h
            fd = (lp - lm) / (2 * h)
            assert abs(fd - W.grad[i, j].item()) <= 1e-5 * max(1.0, abs(fd)), (k, i, j, fd, W.grad[i, j].item())
