"""The checker of the training torso-SR field (oracle/torso_sr_train.py) against tests/golden/train_torso_sr.npz -- the reference's own
RADNeRFTorsowithSR.forward_torso + backward in parts (a) head-aware with an image, (b) image=None, (c) no head-aware encoder and no
code -- and against central finite differences in float64.  CPU only."""
import os

import numpy as np
import pytest
import torch

from oracle import ops
from oracle import torso_sr_train as tst

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_torso_sr.npz")


@pytest.fixture(scope="module", autouse=True)
def _build():
    ops.build()


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize("part", list(tst.PARTS))
def test_oracle_against_reference_golden(part):
    z = np.load(GOLDEN)
    hp = tst.golden_hparams(part)
    state = tst.golden_state(hp)
    ha = bool(hp["torso_head_aware"])
    has_code = hp["torso_individual_embedding_dim"] > 0
    pts = tst.golden_points()
    image, ws = (pts["image"], pts["weights_sum"]) if part == "a" else (None, None)
    idx = torch.from_numpy(z["table_sample_idx"])
    for dtype, pre, bar in ((torch.float32, "grad", 1e-5), (torch.float64, "grad64", 1e-6)):   # grad64 is stored in fp32
        p = tst.torso_sr_params(state, ha, dtype)
        codes = state["torso_individual_codes"].to(dtype).clone().requires_grad_(True) if has_code else None
        a, c, dx = tst.torso_sr_forward(p, hp, pts["x"], tst.golden_lm68(), codes[[tst.GOLDEN_INDEX]] if has_code else None, image, ws)
        tst.linear_loss(a, c, dx, pts).backward()
        if dtype == torch.float32:
            for k, o in (("alpha", a), ("color", c), ("deform", dx)):
                assert _rel(o.detach(), z[f"{part}.{k}"]) <= 1e-5, k
        for k in tst.trainable(ha):
            got = p[k].grad[idx] if k == "torso_embedder.embeddings" else p[k].grad
            key = f"{part}.{pre}.table_sample" if k == "torso_embedder.embeddings" else f"{part}.{pre}.{k}"
            assert _rel(got, z[key]) <= bar, (dtype, k, _rel(got, z[key]))
        if has_code:
            assert _rel(codes.grad[tst.GOLDEN_INDEX], z[f"{part}.{pre}.code"]) <= bar


@pytest.mark.parametrize("part", ["a", "c"])
def test_oracle_against_finite_differences(part):
    """float64 autograd gradients against central differences, at 64 points away from ties, for a few entries of every dense
    parameter: the canonical net with the full linear loss; the deform net and head_color_weights_encoder with the loss on dx alone
    (their path through the grid passes the fp32 clamp output, as in the reference, which finite differences cannot resolve)."""
    hp = tst.golden_hparams(part)
    state = tst.golden_state(hp)
    ha = bool(hp["torso_head_aware"])
    pts = tst.golden_points(256, seed=77)
    trace = {}
    p = tst.torso_sr_params(state, ha, torch.float64)
    image, ws = (pts["image"], pts["weights_sum"]) if part == "a" else (None, None)
    lm68 = tst.golden_lm68()
    tst.torso_sr_forward(p, hp, pts["x"], lm68, None if not hp["torso_individual_embedding_dim"] else state["torso_individual_codes"][:1].double(),
                         image, ws, trace)
    keep = torch.nonzero(~tst.tie_mask(trace, eps=1e-4)).reshape(-1)[:64]
    pts = {k: v[keep] for k, v in pts.items()}
    image, ws = (pts["image"], pts["weights_sum"]) if part == "a" else (None, None)
    code = state["torso_individual_codes"][:1].double() if hp["torso_individual_embedding_dim"] else None

    dx_only = {**pts, "ca": torch.zeros_like(pts["ca"]), "cc": torch.zeros_like(pts["cc"])}
    g = torch.Generator().manual_seed(5)
    h = 1e-6
    for k in tst.trainable(ha):
        if k == "torso_embedder.embeddings":
            continue
        coef = pts if k.startswith("torso_canonicial_net") else dx_only

        def loss(p):
            return tst.linear_loss(*tst.torso_sr_forward(p, hp, pts["x"], lm68, code, image, ws), coef)

        p = tst.torso_sr_params(state, ha, torch.float64)
        loss(p).backward()
        w = p[k]
        for _ in range(3):
            i = int(torch.randint(w.numel(), (1,), generator=g))
            with torch.no_grad():
                q = {kk: (v.detach().clone() if torch.is_tensor(v) and v.dtype == torch.float64 else v) for kk, v in p.items()}
                q[k].view(-1)[i] += h
                lp = loss(q).item()
                q[k].view(-1)[i] -= 2 * h
                lm = loss(q).item()
            fd = (lp - lm) / (2 * h)
            an = w.grad.view(-1)[i].item()
            assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (k, i, fd, an)
