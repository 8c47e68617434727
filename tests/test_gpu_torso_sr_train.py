"""The trainable torso-SR field on the GPU (gfpp.h section I: RADNeRFTorsowithSR.forward_torso in training mode, fused fp32 forward
and backward, csrc/torso_train_kernel.cu):
  * the training forward is bit-identical to the render epilogue's (gfpp_torso_sr_composite) alpha and deform at its masked pixels;
  * gradients against the float64 autograd oracle (oracle/torso_sr_train.py) for several M and configurations (head-aware with and
    without an image, no head-aware encoder and no code), no further from float64 than the fp32 arithmetic of the reference;
  * against tests/golden/train_torso_sr.npz: the reference's own forward_torso + backward, parts (a), (b), (c);
  * determinism, the gradient targets (the code row, head_color_weights_encoder; sr_net and the head get none), the table gradient
    (which the host-side field this replaces never produced), and three Adam steps against an eager fp32 restatement.
"""
import copy
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
from oracle import ops
from oracle import torso_sr_train as tst

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_torso_sr.npz")
FLOOR = 2e-4             # the bar's floor, relative to max|float64 gradient|: the fp32 level of this field away from ties (the fp32
                         # checker, i.e. the reference's arithmetic, is measured up to 2.4e-4 from float64; the first layers sum ~200
                         # inputs of magnitude up to ~10)
FWD_REL = 1e-5           # forward outputs against the reference golden
ADAM_LOSS_REL = 1e-3     # 3 Adam steps: loss, against the eager fp32 restatement (measured 2.0e-5)
FIRST_STEP_REL = 2e-3   # first-step gradients, fused against eager fp32, relative to max|eager|


def _model(part):
    hp = tst.golden_hparams(part)
    state = tst.golden_state(hp)
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(state, strict=False)
    return m.cuda().train(), hp, state


@pytest.fixture(scope="module")
def models():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    ops.build()
    return {p: _model(p) for p in tst.PARTS}


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _inputs(part, pts):
    return (pts["image"], pts["weights_sum"]) if part == "a" else (None, None)


def _gpu_grads(m, part, pts, lm68, index=tst.GOLDEN_INDEX):
    """forward_torso + backward of the linear loss on the GPU; returns outputs and gradients (CPU), keyed by state-dict name."""
    m.zero_grad(set_to_none=True)
    image, ws = _inputs(part, pts)
    c = m.torso_individual_codes[torch.tensor([index], device="cuda")] if m.torso_individual_embedding_dim else None
    a, col, dx = m.forward_torso(pts["x"].cuda(), None, c, None if image is None else image.cuda(), None if ws is None else ws.cuda(),
                                 lm68=lm68.cuda())
    tst.linear_loss(a, col, dx, {k: v.cuda() for k, v in pts.items()}).backward()
    torch.cuda.synchronize()
    params = dict(m.named_parameters())
    g = {k: params[k].grad.cpu() for k in tst.trainable(m.torso_head_aware)}
    if m.torso_individual_embedding_dim:
        g["code"] = params["torso_individual_codes"].grad[index].cpu()
    return (a.detach().cpu(), col.detach().cpu(), dx.detach().cpu()), g


def _oracle_grads(hp, state, part, pts, lm68, dtype, trace=None):
    ha = bool(hp["torso_head_aware"])
    p = tst.torso_sr_params(state, ha, dtype)
    has_code = hp["torso_individual_embedding_dim"] > 0
    codes = state["torso_individual_codes"].to(dtype).clone().requires_grad_(True) if has_code else None
    image, ws = _inputs(part, pts)
    o = tst.torso_sr_forward(p, hp, pts["x"], lm68, codes[[tst.GOLDEN_INDEX]] if has_code else None, image, ws, trace)
    tst.linear_loss(*o, pts).backward()
    g = {k: p[k].grad for k in tst.trainable(ha)}
    if has_code:
        g["code"] = codes.grad[tst.GOLDEN_INDEX]
    return tuple(t.detach() for t in o), g


def _golden_fp32_err(part):
    """The reference's own fp32 error against float64 in golden part `part`, per gradient, relative to max|float64|."""
    z = np.load(GOLDEN)
    pre = f"{part}.grad."
    return {k[len(pre):]: _rel(z[k], z[f"{part}.grad64." + k[len(pre):]]) for k in z.files if k.startswith(pre) and "table" not in k}


def test_training_forward_is_bit_identical_to_the_composite(models):
    """c = torso_individual_codes[0], one lm68 row, image / weights_sum at the masked pixels of a one-frame gfpp_torso_sr_composite:
    the training forward's alpha and deform equal the composite's torso_alpha_map and torso_deform bit for bit."""
    m, hp, _ = models["a"]
    g = torch.Generator().manual_seed(11)
    R = 128
    N = R * R
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, R), torch.linspace(-1, 1, R), indexing="ij")
    bg_coords = torch.stack([xs, ys], -1).reshape(N, 2).cuda()
    ws = torch.rand(1, N, generator=g).cuda()
    image = (torch.rand(1, N, 3, generator=g).cuda() * ws.unsqueeze(-1)).contiguous()
    lm68 = tst.golden_lm68().cuda()
    with torch.no_grad():
        m.density_grid_torso.copy_(torch.rand(m.grid_size ** 2, generator=g).cuda())
    m.mean_density_torso = 0.5
    tr = m.torso_composite_native(image, ws, lm68, bg_coords)
    mask = tr["torso_alpha_map"][0] != 0
    assert 0 < int(mask.sum()) < N and int(tr["torso_pixels"][0]) == int(mask.sum())
    c = m.torso_individual_codes[0]
    a, col, dx = m.forward_torso(bg_coords[mask], None, c, image[0][mask], ws[0][mask].unsqueeze(-1), lm68=lm68)
    assert a.requires_grad and a.dtype == torch.float32
    assert torch.equal(a.detach().view(-1), tr["torso_alpha_map"][0][mask])
    assert torch.equal(dx.detach(), tr["deform"][0][mask])
    with torch.autocast("cuda", dtype=torch.float16):
        a2, _, _ = m.forward_torso(bg_coords[mask], None, c, image[0][mask], ws[0][mask].unsqueeze(-1), lm68=lm68)
    assert a2.dtype == torch.float32 and torch.equal(a2.detach(), a.detach())
    with torch.no_grad():
        a3, _, _ = m.forward_torso(bg_coords[mask], None, c, image[0][mask], ws[0][mask].unsqueeze(-1), lm68=lm68)
    assert not a3.requires_grad and torch.equal(a3, a.detach())


CASES = [("a", M) for M in (1, 127, 128, 129, 3000, 65536, 262144)] + [("b", 129), ("b", 3000), ("c", 129), ("c", 3000)]


@pytest.mark.parametrize("part,M", CASES, ids=[f"{p}-{M}" for p, M in CASES])
def test_gradients_against_float64(models, part, M):
    """Part a: head-aware with image and code; b: image=None; c: no head-aware encoder, no code.  Each gradient is no further from
    float64 than max(2 x the reference's own fp32 error (golden), 2 x the fp32 checker's at these points, FLOOR x max|grad|).  Points
    within 1e-4 of a ReLU / LeakyReLU kink or within 1e-6 of a clamp bound or of a grid cell boundary are excluded (oracle
    tie_mask; counted and printed)."""
    m, hp, state = models[part]
    lm68 = tst.golden_lm68()
    pts = tst.golden_points(M + 64 + M // 4, seed=1000 + M)
    trace = {}
    _oracle_grads(hp, state, part, pts, lm68, torch.float64, trace)
    keep = ~tst.tie_mask(trace)
    n_tie = int((~keep).sum())
    idx = torch.nonzero(keep).reshape(-1)[:M]
    pts = {k: v[idx] for k, v in pts.items()}
    out, gg = _gpu_grads(m, part, pts, lm68)
    o64, g64 = _oracle_grads(hp, state, part, pts, lm68, torch.float64)
    _, g32 = _oracle_grads(hp, state, part, pts, lm68, torch.float32)
    ref_err = _golden_fp32_err(part)
    e_fwd = max((a.double() - b).abs().max().item() for a, b in zip(out, o64))
    print(f"\n{part} M={M}: {n_tie} points at a tie, a clamp bound or a grid cell boundary excluded; forward max abs error {e_fwd:.2e}")
    assert e_fwd <= 1e-5
    for k in g64:
        e, e32 = _rel(gg[k], g64[k]), _rel(g32[k], g64[k])
        bar = max(2 * ref_err.get(k, 0.0), 2 * e32, FLOOR)
        print(f"  {k}: libgfpp {e:.2e}, fp32 checker {e32:.2e}, reference (golden) {ref_err.get(k, float('nan')):.2e}; bar {bar:.2e}")
        assert e <= bar, (k, e, bar)


@pytest.mark.parametrize("part", list(tst.PARTS))
def test_against_reference_golden(models, part):
    """forward_torso + backward at the golden's points against the reference's own (tests/golden/train_torso_sr.npz).  The forward
    outputs are compared directly.  For the gradients, the contributions of the points within the tie margins (oracle tie_mask) are
    removed from both sides -- from the golden with the fp32 checker, whose arithmetic equals the reference's bit for bit
    (tests/test_oracle_torso_sr_train.py), from libgfpp with its own gradient at those points -- because fp32 in another summation
    order may take the other branch there; the remaining gradients are held to the float64 bar of the reference itself."""
    m, hp, state = models[part]
    z = np.load(GOLDEN)
    pts, lm68 = tst.golden_points(), tst.golden_lm68()
    out, gg = _gpu_grads(m, part, pts, lm68)
    for k, o in zip(("alpha", "color", "deform"), out):
        e = _rel(o, z[f"{part}.{k}"])
        print(f"golden ({part}) {k}: rel {e:.2e}")
        assert e <= FWD_REL, (k, e)
    trace = {}
    _oracle_grads(hp, state, part, pts, lm68, torch.float64, trace)
    tie = torch.nonzero(tst.tie_mask(trace)).reshape(-1)
    sub = {k: v[tie] for k, v in pts.items()}
    _, gg_t = _gpu_grads(m, part, sub, lm68)
    _, g32_t = _oracle_grads(hp, state, part, sub, lm68, torch.float32)
    _, g64_t = _oracle_grads(hp, state, part, sub, lm68, torch.float64)
    idx = torch.from_numpy(z["table_sample_idx"])
    print(f"golden ({part}): {tie.numel()} of {tst.GOLDEN_M} points within the tie margins removed")
    for k in gg:
        sel = (lambda t: t[idx]) if k == "torso_embedder.embeddings" else (lambda t: t)
        key = "table_sample" if k == "torso_embedder.embeddings" else k
        ref = torch.from_numpy(z[f"{part}.grad.{key}"]).double() - sel(g32_t[k]).double()
        ref64 = torch.from_numpy(z[f"{part}.grad64.{key}"]).double() - sel(g64_t[k]).double()
        got = sel(gg[k]).double() - sel(gg_t[k]).double()
        e, e_ref = _rel(got, ref64), _rel(ref, ref64)
        print(f"golden ({part}) {k}: to float64 libgfpp {e:.2e}, reference {e_ref:.2e}; to the reference {_rel(got, ref):.2e}")
        assert e <= max(2 * e_ref, FLOOR), (k, e, e_ref)


def test_deterministic_and_gradient_targets(models):
    """Two runs give bit-identical weight, bias and code gradients; only row `index` of the codes, the torso field and
    head_color_weights_encoder get gradients; sr_net and the head none.  The table gradient is non-zero and matches the float64
    oracle: the host-side field this path replaces returned an untracked grid encoding (no table gradient at all)."""
    m, hp, state = models["a"]
    pts = tst.golden_points(100000, seed=7)
    lm68 = tst.golden_lm68()
    _, g1 = _gpu_grads(m, "a", pts, lm68)
    full = m.torso_individual_codes.grad.detach().clone()
    _, g2 = _gpu_grads(m, "a", pts, lm68)
    for k in g1:
        if k != "torso_embedder.embeddings":
            assert torch.equal(g1[k], g2[k]), k
    assert torch.nonzero(full.abs().sum(-1)).reshape(-1).tolist() == [tst.GOLDEN_INDEX]
    for k in tst.HEAD_AWARE:
        assert g1[k].abs().sum() > 0, k
    trained = set(tst.trainable(True)) | {"torso_individual_codes"}
    for k, p in m.named_parameters():
        if k not in trained:
            assert p.grad is None, k
    tab = g1["torso_embedder.embeddings"]
    assert tab.abs().sum() > 0
    small = {k: v[:3064] for k, v in pts.items()}
    trace = {}
    _oracle_grads(hp, state, "a", small, lm68, torch.float64, trace)
    small = {k: v[~tst.tie_mask(trace)][:3000] for k, v in small.items()}
    _, gs = _gpu_grads(m, "a", small, lm68)
    _, g64 = _oracle_grads(hp, state, "a", small, lm68, torch.float64)
    e = _rel(gs["torso_embedder.embeddings"], g64["torso_embedder.embeddings"])
    _, g32 = _oracle_grads(hp, state, "a", small, lm68, torch.float32)
    e32 = _rel(g32["torso_embedder.embeddings"], g64["torso_embedder.embeddings"])
    print(f"table gradient at 3000 points away from ties: rel {e:.2e} to float64 (fp32 checker {e32:.2e})")
    assert e <= max(2 * e32, FLOOR)


def test_m0_and_guards(models):
    m, _, _ = models["a"]
    c = m.torso_individual_codes[torch.tensor([1], device="cuda")]
    lm68 = tst.golden_lm68().cuda()
    a, col, dx = m.forward_torso(torch.zeros(0, 2, device="cuda"), None, c, None, None, lm68=lm68)
    (a.sum() + col.sum() + dx.sum()).backward()
    assert a.shape == (0, 1) and col.shape == (0, 3) and dx.shape == (0, 2)
    x = torch.zeros(4, 2, device="cuda")
    for kw in ({"x": x.clone().requires_grad_(True)}, {"image": torch.zeros(4, 3, device="cuda", requires_grad=True)},
               {"lm68": lm68.clone().requires_grad_(True)}):
        args = {"x": x, "image": torch.zeros(4, 3, device="cuda"), "weights_sum": torch.zeros(4, 1, device="cuda"), "lm68": lm68, **kw}
        with pytest.raises(NotImplementedError):
            m.forward_torso(args["x"], None, c, args["image"], args["weights_sum"], lm68=args["lm68"])
    with pytest.raises(ValueError):
        m.forward_torso(x, None, c, torch.zeros(4, 3, device="cuda"), None, lm68=lm68)


def test_three_adam_steps_against_eager_fp32(models):
    """Three Adam steps of the README recipe (field step + the task's torso loss: MSE on torso_rgb_map, alpha entropy,
    lambda_torso_deform * |deform|) on the fused field and on the eager fp32 restatement (F.linear over train_ops.grid_encode), on
    pixels away from the tie margins: the first step's gradients and the three losses agree; the parameter drift is printed."""
    base, hp, state = models["a"]
    g = torch.Generator().manual_seed(3)
    N = 64 * 64
    bg_coords = torch.rand(N, 2, generator=g) * 2 - 1
    ws = torch.rand(N, 1, generator=g)
    image = torch.rand(N, 3, generator=g) * ws
    gt = torch.rand(N, 3, generator=g).cuda()
    lm68 = tst.golden_lm68()
    trace = {}
    tst.torso_sr_forward(tst.torso_sr_params(state, True, torch.float64), hp, bg_coords, lm68,
                         state["torso_individual_codes"][[tst.GOLDEN_INDEX]].double(), image, ws, trace)
    mask = ((torch.rand(N, generator=g) < 0.6) & ~tst.tie_mask(trace)).cuda()
    bg_coords, ws, image, lm68 = bg_coords.cuda(), ws.cuda(), image.cuda(), lm68.cuda()
    bg = torch.ones(1, 3, device="cuda")
    index = torch.tensor([tst.GOLDEN_INDEX], device="cuda")
    torch.backends.cuda.matmul.allow_tf32 = False
    names = [f"torso_deform_net.net.{i}.weight" for i in range(3)] + [f"torso_canonicial_net.net.{i}.weight" for i in range(3)] + \
            ["torso_embedder.embeddings"] + [f"head_color_weights_encoder.{i}.{k}" for k in ("weight", "bias") for i in (0, 2, 4)] + \
            ["torso_individual_codes"]
    res = {}
    for leg in ("fused", "eager"):
        m = copy.deepcopy(base)
        params = train_ops.torso_sr_params(m) + [m.torso_individual_codes]
        opt = torch.optim.Adam(params, lr=5e-3, betas=(0.9, 0.99), eps=1e-15)
        losses, first = [], None
        for step in range(3):
            opt.zero_grad(set_to_none=True)
            c = m.torso_individual_codes[index]
            if leg == "fused":
                a, col, dx = m.forward_torso(bg_coords[mask], None, c, image[mask], ws[mask], lm68=lm68)
            else:
                a, col, dx = tst.eager_torso_sr(m, tst.model_params(m), bg_coords[mask], lm68, c, image[mask], ws[mask], train_ops.grid_encode)
            loss = tst.composite_and_loss(a, col, dx, mask, bg, gt)
            loss.backward()
            if step == 0:
                first = [p.grad.detach().clone() for p in params]
            opt.step()
            losses.append(loss.item())
        res[leg] = (losses, first, [p.detach().clone() for p in params])
    for i, (lf, le) in enumerate(zip(res["fused"][0], res["eager"][0])):
        print(f"step {i}: loss fused {lf:.6e}, eager {le:.6e}")
        assert abs(lf - le) <= ADAM_LOSS_REL * abs(le), (i, lf, le)
    for name, gf, ge, pf, pe in zip(names, res["fused"][1], res["eager"][1], res["fused"][2], res["eager"][2]):
        e = _rel(gf, ge)
        drift = ((pf - pe).norm() / pe.norm().clamp_min(1e-30)).item()
        print(f"  {name}: first-step gradient rel {e:.2e}; after 3 steps, relative L2 fused - eager {drift:.2e}")
        assert e <= FIRST_STEP_REL, (name, e)
