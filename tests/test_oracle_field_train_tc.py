"""The rounding oracle of the tensor-core training field (oracle/field_train_tc.py): with rounding off it is oracle/field_train.py bit
for bit, outputs, gradients and trace; with rounding on its outputs and gradients on the inputs of tests/golden/train_head.npz stay
within the bars the GPU tests hold the kernels to (tests/test_gpu_field_train_tc.py).  The output-gradient scale rule is the kernels'
block_scale: the exponent per 128-point block, the per-call rule when one block holds the call, identical results on seeded random
inputs, faint tiles that keep their bits where the per-call rule flushes them, and exact loss scaling."""
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


def test_trace_is_the_relu_inputs(case):
    """trace["relu_pre"]: five [N,128] pre-activations; with rounding off they are oracle/field_train.py's own, bit for bit."""
    sc, x, d, cond, _ = case
    p, code = ft.field_params(sc.state), sc.state["individual_embeddings"][2]
    t_off, t_on, t_ref = {}, {}, {}
    ftc.field_forward(p, sc.hparams, x, d, cond, code, rounding=False, trace=t_off)
    ftc.field_forward(p, sc.hparams, x, d, cond, code, trace=t_on)
    ft.field_forward(p, sc.hparams, x, d, cond, code, trace=t_ref)
    assert len(t_on["relu_pre"]) == 5 and all(t.shape == (x.shape[0], 128) for t in t_on["relu_pre"])
    assert all(torch.equal(a, b) for a, b in zip(t_off["relu_pre"], t_ref["relu_pre"]))
    assert not all(torch.equal(a, b) for a, b in zip(t_on["relu_pre"], t_ref["relu_pre"]))


# ------------------------------------------------------------------------------------------------ the per-tile scale rule
def _per_call(g):
    """The scale rule with one power of two per call: g's largest magnitude to [256, 512)."""
    m = float(g.abs().max())
    if not (0.0 < m < float("inf")):
        return ftc._r16(g)
    s = 2.0 ** (8 - int(np.floor(np.log2(m))))
    return ftc._r16(g * s) / s


def _kernel_exponent(m):
    """block_scale's k for a float32 largest magnitude m, from its biased exponent bits as the kernel computes it."""
    if not (m > 0 and np.isfinite(m)):
        return 0
    bits = int(np.array(m, dtype=np.float32).view(np.int32))
    return min(126, max(-126, 135 - ((bits >> 23) & 255)))


def test_block_exponents_are_block_scale():
    mags = [1.0, 255.0, 256.0, 511.99, 512.0, 3e-5, 2.0 ** -126, 2.0 ** -140, 1e-45, 2.0 ** 100, 3e38, 0.0, float("inf")]
    g = torch.zeros(128 * len(mags) - 5, 7)
    for i, m in enumerate(mags):
        g[128 * i + (i % 100), i % 7] = -m if i % 2 else m
        g[128 * i + 3, 0] = float("nan") if i == 2 else g[128 * i + 3, 0]   # NaN is not the largest magnitude (fmaxf drops it)
    k = ftc.block_exponents(g)
    want = [_kernel_exponent(np.float32(m)) for m in mags]
    assert k.tolist() == want, (k.tolist(), want)
    scaled = torch.ldexp(torch.tensor(mags[:5]), k[:5])
    assert bool(((scaled >= 256) & (scaled < 512)).all())


def test_per_tile_rule_with_one_block_is_the_per_call_rule(monkeypatch):
    g = torch.randn(3001, 128, generator=torch.Generator().manual_seed(3)) * torch.logspace(-6, 3, 3001).unsqueeze(1)
    per_tile = ftc._r16_scaled(g)
    monkeypatch.setattr(ftc, "TILE", 1 << 30)
    assert torch.equal(ftc._r16_scaled(g), _per_call(g))
    assert not torch.equal(per_tile, _per_call(g))   # the magnitudes here span nine decades: the tiles differ


@pytest.fixture(scope="module")
def seeded():
    """tests/test_gpu_field_train_tc.py's 3 001 points (seed 7, uniform in aabb_train) and upstream gradients, with the golden's
    conditioning vector."""
    ops.build()
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_head.npz"))
    sc = scn.Scene(H=32, W=32, T=4, torso=False, density_scale=8.0)
    g = torch.Generator().manual_seed(7)
    M = 3001
    lo, hi = sc.state["aabb_train"][:3], sc.state["aabb_train"][3:]
    x = lo + (hi - lo) * torch.rand(M, 3, generator=g)
    d = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=-1)
    up = [torch.randn(M, generator=g), torch.randn(M, 3, generator=g), torch.randn(M, 3, generator=g)]
    return sc, x, d, torch.from_numpy(G["cond_feat"]), up


def test_per_tile_and_per_call_agree_on_seeded_inputs(seeded, monkeypatch):
    """Tiles of random points have largest magnitudes within a few binades of each other: the two rules round alike."""
    out, g = _run(ftc.field_forward, seeded)
    monkeypatch.setattr(ftc, "TILE", 1 << 30)
    out1, g1 = _run(ftc.field_forward, seeded)
    assert all(torch.equal(a, b) for a, b in zip(out, out1))
    for k in g:
        assert torch.equal(g[k], g1[k]), k


def _spread(case, faint, tiles=None):
    """case with the upstream gradients of every other 128-point tile (odd tiles) times `faint`; tiles: keep only the rows of the
    loud ("loud") or faint ("faint") tiles' upstream."""
    sc, x, d, cond, up = case
    odd = (torch.arange(x.shape[0]) // 128) % 2 == 1
    f = torch.where(odd, torch.tensor(faint), torch.tensor(1.0))
    if tiles == "loud":
        f = torch.where(odd, torch.tensor(0.0), f)
    elif tiles == "faint":
        f = torch.where(odd, f, torch.tensor(0.0))
    return sc, x, d, cond, [u * f.view(-1, *([1] * (u.dim() - 1))) for u in up]


def _run64(case):
    sc, x, d, cond, up = case
    p = ft.field_params(sc.state, torch.float64)
    c = cond.clone().double().requires_grad_(True)
    code = sc.state["individual_embeddings"][2].clone().double().requires_grad_(True)
    out = ft.field_forward(p, sc.hparams, x, d.double(), c, code)
    sum((o * u.double()).sum() for o, u in zip(out, up)).backward()
    return {k: p[k].grad for k in ft.TRAINABLE}


FAINT = 2.0 ** -40


def test_faint_tiles_keep_their_bits(seeded, monkeypatch):
    """Upstream gradients with alternate tiles 2^-40 times fainter.  Position-table entries that only faint-tile points reach: the
    per-tile rule gives them exactly 2^-40 times what the same points give at full strength, close to float64; the per-call rule
    (one power of two from the loud tiles) rounds the faint tiles' dY to zero and leaves those entries at exactly 0."""
    sc, x, d, cond, up = seeded
    n = 1024                                            # eight tiles, four of them faint
    case = (sc, x[:n], d[:n], cond, [u[:n] for u in up])
    key = "position_embedder.embeddings"
    loud64, faint64 = _run64(_spread(case, FAINT, "loud"))[key], _run64(_spread(case, FAINT, "faint"))[key]
    only = (faint64 != 0).any(1) & (loud64 == 0).all(1)
    assert int(only.sum()) > 1000, int(only.sum())
    _, g = _run(ftc.field_forward, _spread(case, FAINT))
    _, g_full = _run(ftc.field_forward, _spread(case, 1.0))
    ref = _run64(_spread(case, FAINT))[key]
    t, t_full = g[key][only], g_full[key][only]
    l2 = ((t.double() - ref[only]).norm() / ref[only].norm()).item()
    print(f"per-tile rule: {int(only.sum())} position-table entries reached only by faint tiles, {int((t != 0).any(1).sum())} non-zero, "
          f"rel L2 to float64 {l2:.2e}")
    assert torch.equal(t, t_full * FAINT)
    assert bool(((t != 0) | (ref[only] == 0)).all()) and l2 <= GRAD_L2_UPSTREAM
    assert all(bool(torch.isfinite(v).all()) for v in g.values())
    monkeypatch.setattr(ftc, "TILE", 1 << 30)
    _, g1 = _run(ftc.field_forward, _spread(case, FAINT))
    print(f"per-call rule: max |entry| of those entries {g1[key][only].abs().max().item():.1e}")
    assert float(g1[key][only].abs().max()) == 0.0


def test_loss_scale_is_exact(seeded):
    """Upstream gradients times 2^k: every gradient of the per-tile oracle times exactly 2^k (each block's power of two absorbs it)."""
    _, g = _run(ftc.field_forward, seeded)
    for k in (-20, 12):
        sc, x, d, cond, up = seeded
        _, gk = _run(ftc.field_forward, (sc, x, d, cond, [u * 2.0 ** k for u in up]))
        for name in g:
            assert torch.equal(gk[name], g[name] * 2.0 ** k), (k, name)


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
