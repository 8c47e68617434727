"""The rounding oracle of the tensor-core training field (oracle/field_train_tc.py): with rounding off it is oracle/field_train.py bit
for bit, outputs and gradients; with rounding on its outputs and gradients on the inputs of tests/golden/train_head.npz stay within
the bars the GPU tests hold the kernels to (tests/test_gpu_field_train_tc.py)."""
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from oracle import field_train as ft
from oracle import field_train_tc as ftc
from oracle import ops

FWD_ABS = 1e-4           # colour / ambient, absolute (measured 1.9e-5 / 2.4e-5)
FWD_SIGMA_REL = 1.5e-3   # sigma, relative to the largest sigma (measured 4.1e-4)
# Gradients, relative L2 against the fp32 oracle.  The field amplifies operand rounding (tools/error_budget.py): an fp16-rounded
# activation moves the ambient coordinates across cells of the fine ambient-grid levels, where dy_dx jumps, and flips ReLUs at ties.
GRAD_L2 = 0.15           # sigma and colour nets, ambient table, code (measured 5.2e-4 to 5.9e-2)
GRAD_L2_UPSTREAM = 0.4   # what comes through the ambient grid's input gradient (measured 1.16e-1 to 1.38e-1)
UPSTREAM = ("ambient_net.net.0.weight", "ambient_net.net.1.weight", "ambient_net.net.2.weight", "position_embedder.embeddings", "cond")


@pytest.fixture(scope="module")
def case():
    ops.build()
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_head.npz"))
    sc = scn.Scene(H=32, W=32, T=4, torso=False, density_scale=8.0)
    x = torch.from_numpy(G["position"])
    x = x[x.abs().sum(1) > 0][:2000]
    g = torch.Generator().manual_seed(5)
    d = torch.nn.functional.normalize(torch.randn(x.shape[0], 3, generator=g), dim=-1)
    up = [torch.randn(x.shape[0], generator=g), torch.randn(x.shape[0], 3, generator=g), torch.randn(x.shape[0], 3, generator=g)]
    return sc, x, d, torch.from_numpy(G["cond_feat"]), up


def _run(fwd, case):
    sc, x, d, cond, up = case
    p = ft.field_params(sc.state)
    c = cond.clone().requires_grad_(True)
    code = sc.state["individual_embeddings"][2].clone().requires_grad_(True)
    out = fwd(p, sc.hparams, x, d, c, code)
    sum((o * u).sum() for o, u in zip(out, up)).backward()
    grads = {k: p[k].grad for k in ft.TRAINABLE}
    grads.update(cond=c.grad, code=code.grad)
    return [o.detach() for o in out], grads


def test_rounding_off_is_the_fp32_oracle(case):
    out, g = _run(lambda *a: ftc.field_forward(*a, rounding=False), case)
    ref, r = _run(ft.field_forward, case)
    for a, b in zip(out, ref):
        assert torch.equal(a, b)
    for k in r:
        assert torch.equal(g[k], r[k]), k


def test_rounding_on_stays_within_the_bars(case):
    out, g = _run(ftc.field_forward, case)
    ref, r = _run(ft.field_forward, case)
    e = [(out[0] - ref[0]).abs().max().item() / ref[0].abs().max().item(), (out[1] - ref[1]).abs().max().item(),
         (out[2] - ref[2]).abs().max().item()]
    print(f"rounding oracle vs fp32 oracle: sigma rel {e[0]:.2e}, colour abs {e[1]:.2e}, ambient abs {e[2]:.2e}")
    assert e[0] <= FWD_SIGMA_REL and e[1] <= FWD_ABS and e[2] <= FWD_ABS
    assert max(e) > 0
    bad = []
    for k in r:
        l2 = ((g[k] - r[k]).norm() / r[k].norm()).item()
        print(f"grad {k}: rel L2 {l2:.2e}")
        if l2 > (GRAD_L2_UPSTREAM if k in UPSTREAM else GRAD_L2):
            bad.append((k, l2))
    assert not bad, bad
