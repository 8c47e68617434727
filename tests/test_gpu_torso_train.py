"""The trainable torso field on the GPU (gfpp.h section H: RADNeRFTorso.forward_torso in training mode, fused fp32 forward and
backward, csrc/torso_train_kernel.cu):
  * the training-mode forward is bit-identical to the eval-mode (packed) query;
  * gradients against the float64 autograd oracle (oracle/torso_train.py) at random points for several M, no further from float64
    than the reference's own fp32 result;
  * against tests/golden/train_torso.npz: (a) the reference's own forward_torso + backward, (b) its torso training step, restated
    on libgfpp (oracle/torso_train.gfpp_train_step: the README recipe);
  * determinism, the code row, and three Adam steps against an eager fp32 restatement.
"""
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.renderer import RADNeRFTorso
from oracle import ops
from oracle import torso_train as tt

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_torso.npz")
WEIGHTS = tt.TRAINABLE[:6]
FLOOR = 1e-5             # the bar's floor, relative to max|float64 gradient|
FWD_REL = 1e-5           # forward outputs against the reference golden (fp32 rounding of the same arithmetic)
STEP_OUT = 1e-5          # training-step maps against golden (b)
FIRST_STEP_REL = 5e-4    # first-step gradients against the eager fp32 restatement (both are ~1e-4 from float64 on the deform net)
ADAM_LOSS_REL = 1e-3     # 3 Adam steps: loss (measured 1.4e-4; the eager leg's table scatter order varies from run to run)
ADAM_PARAM_REL = 5e-2    # 3 Adam steps: parameters, relative L2 (measured 9.8e-3: Adam turns noise-level gradients into full steps)


@pytest.fixture(scope="module")
def setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    ops.build()
    sc = tt.golden_scene()
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = tt.GOLDEN_DS
    m.mlp_precision = "fp32"
    m = m.cuda().train()
    fi = sc.frame_inputs(tt.GOLDEN_FRAME)
    return {"sc": sc, "model": m, "fi": fi, "pose6": fi["poses"], "index": torch.tensor([tt.GOLDEN_INDEX])}


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _gpu_grads(m, x, pose6, index, coef):
    """forward_torso + backward of sum(alpha*ca) + sum(color*cc) + sum(dx*cd) on the GPU; returns outputs and gradients (CPU)."""
    m.zero_grad(set_to_none=True)
    a, c, dx = m.forward_torso(x.cuda(), pose6.cuda(), m.torso_individual_codes[index.cuda()])
    ((a * coef[0].cuda()).sum() + (c * coef[1].cuda()).sum() + (dx * coef[2].cuda()).sum()).backward()
    torch.cuda.synchronize()
    params = dict(m.named_parameters())
    g = {k: params[k].grad.cpu() for k in tt.TRAINABLE}
    g["code"] = params["torso_individual_codes"].grad[int(index)].cpu()
    return (a.detach().cpu(), c.detach().cpu(), dx.detach().cpu()), g, params["torso_individual_codes"].grad.cpu()


def _oracle_grads(sc, x, pose6, index, coef, dtype, trace=None):
    p = tt.torso_params(sc.state, dtype)
    codes = sc.state["torso_individual_codes"].to(dtype).clone().requires_grad_(True)
    a, c, dx = tt.torso_forward(p, sc.hparams, x, pose6, codes[index], trace)
    ((a * coef[0].to(dtype)).sum() + (c * coef[1].to(dtype)).sum() + (dx * coef[2].to(dtype)).sum()).backward()
    g = {k: p[k].grad for k in tt.TRAINABLE}
    g["code"] = codes.grad[int(index)]
    return (a.detach(), c.detach(), dx.detach()), g


def _golden_fp32_err(prefix):
    """The reference's own fp32 error against float64 in golden part `prefix`, per gradient, relative to max|float64|."""
    z = np.load(GOLDEN)
    return {k: _rel(z[f"{prefix}.grad.{k}"], z[f"{prefix}.grad64.{k}"]) for k in WEIGHTS + ["code"]}


def test_training_forward_is_bit_identical_to_the_eval_query(setup):
    s = setup
    m = s["model"]
    x = torch.rand(65536, 2, generator=torch.Generator().manual_seed(5)).cuda() * 2 - 1
    c = m.torso_individual_codes[s["index"].cuda()]
    a1, c1, d1 = m.forward_torso(x, s["pose6"].cuda(), c)
    assert a1.requires_grad and a1.dtype == torch.float32
    with torch.autocast("cuda", dtype=torch.float16):
        a3, _, _ = m.forward_torso(x, s["pose6"].cuda(), c)
    m.eval()
    try:
        a2, c2, d2 = m.forward_torso(x, s["pose6"].cuda(), c)
    finally:
        m.train()
    assert not a2.requires_grad
    assert torch.equal(a1.detach(), a2) and torch.equal(c1.detach(), c2) and torch.equal(d1.detach(), d2)
    assert a3.dtype == torch.float32 and torch.equal(a3.detach(), a2)
    with torch.no_grad():
        a4, _, _ = m.forward_torso(x, s["pose6"].cuda(), c)
    assert not a4.requires_grad and torch.equal(a4, a2)


@pytest.mark.parametrize("M", [1, 63, 64, 65, 65536, 262144])
def test_gradients_against_float64(setup, M):
    """Each weight, code and table gradient is no further from float64 than max(2 x the reference's own fp32 error (golden (a), and
    the fp32 checker's -- equal to the reference's arithmetic -- at these points), 1e-5 x max|grad|).  Points within 1e-6 of a ReLU
    tie, of a clamp bound or of a grid cell boundary (where dy_dx jumps) are excluded (counted and printed)."""
    s = setup
    sc = s["sc"]
    g = torch.Generator().manual_seed(1000 + M)
    x = torch.rand(M + 64, 2, generator=g) * 2 - 1
    coef = (torch.randn(M + 64, 1, generator=g), torch.randn(M + 64, 3, generator=g), torch.randn(M + 64, 2, generator=g))
    trace = {}
    _oracle_grads(sc, x, s["pose6"], s["index"], coef, torch.float64, trace)
    keep = ~tt.tie_mask(trace)
    n_tie = int((~keep).sum())
    idx = torch.nonzero(keep).reshape(-1)[:M]
    x, coef = x[idx], tuple(c[idx] for c in coef)
    out, gg, _ = _gpu_grads(s["model"], x, s["pose6"], s["index"], coef)
    o64, g64 = _oracle_grads(sc, x, s["pose6"], s["index"], coef, torch.float64)
    _, g32 = _oracle_grads(sc, x, s["pose6"], s["index"], coef, torch.float32)
    ref_err = _golden_fp32_err("a")
    e_fwd = max((a.double() - b).abs().max().item() for a, b in zip(out, o64))
    print(f"\nM={M}: {n_tie} points at a ReLU tie, a clamp bound or a grid cell boundary excluded; forward max abs error {e_fwd:.2e}")
    assert e_fwd <= 1e-5
    for k in WEIGHTS + ["code", "torso_embedder.embeddings"]:
        e = _rel(gg[k], g64[k])
        e32 = _rel(g32[k], g64[k])
        bar = max(2 * ref_err.get(k, 0.0), 2 * e32, FLOOR)
        print(f"  {k}: libgfpp {e:.2e}, fp32 checker {e32:.2e}, reference (golden) {ref_err.get(k, float('nan')):.2e}; bar {bar:.2e}")
        assert e <= bar, (k, e, bar)


def test_against_reference_golden_a(setup):
    """forward_torso + backward at the golden's points against the reference's own (tests/golden/train_torso.npz part (a))."""
    s = setup
    z = np.load(GOLDEN)
    x = torch.from_numpy(z["a.x"])
    coef = tuple(torch.from_numpy(z[k]) for k in ("a.coef_alpha", "a.coef_color", "a.coef_deform"))
    out, gg, _ = _gpu_grads(s["model"], x, torch.from_numpy(z["pose6"]), s["index"], coef)
    for k, o in zip(("alpha", "color", "deform"), out):
        e = _rel(o, z[f"a.{k}"])
        print(f"golden (a) {k}: rel {e:.2e}")
        assert e <= FWD_REL, (k, e)
    _check_golden_grads(z, "a", gg)


def _check_golden_grads(z, prefix, gg):
    idx = torch.from_numpy(z["table_sample_idx"])
    offsets = tt.golden_scene().state["torso_embedder.offsets"]
    for k in WEIGHTS + ["code"]:
        e = _rel(gg[k], z[f"{prefix}.grad64.{k}"])
        e_ref = _rel(z[f"{prefix}.grad.{k}"], z[f"{prefix}.grad64.{k}"])
        e_g = _rel(gg[k], z[f"{prefix}.grad.{k}"])
        print(f"golden ({prefix}) {k}: to float64 libgfpp {e:.2e}, reference {e_ref:.2e}; to the reference {e_g:.2e}")
        assert e <= max(2 * e_ref, FLOOR), (k, e, e_ref)
    tab = gg["torso_embedder.embeddings"]
    e = _rel(tab[idx], z[f"{prefix}.grad64.table_sample"])
    e_ref = _rel(z[f"{prefix}.grad.table_sample"], z[f"{prefix}.grad64.table_sample"])
    off = offsets.tolist()
    norms = np.asarray([float(tab[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)])
    n64 = np.maximum(z[f"{prefix}.grad64.table_level_norms"], 1e-30)
    en = float(np.max(np.abs(norms - n64) / n64))
    en_ref = float(np.max(np.abs(z[f"{prefix}.grad.table_level_norms"] - n64) / n64))
    print(f"golden ({prefix}) table: sampled entries to float64 libgfpp {e:.2e}, reference {e_ref:.2e}; per-level norms to float64 "
          f"libgfpp {en:.2e}, reference {en_ref:.2e}")
    assert e <= max(2 * e_ref, FLOOR) and en <= max(2 * en_ref, 1e-4), (e, e_ref, en, en_ref)


def test_backward_is_deterministic_and_reaches_only_the_code_row(setup):
    s = setup
    g = torch.Generator().manual_seed(7)
    x = torch.rand(100000, 2, generator=g) * 2 - 1
    coef = (torch.randn(100000, 1, generator=g), torch.randn(100000, 3, generator=g), torch.randn(100000, 2, generator=g))
    _, g1, full1 = _gpu_grads(s["model"], x, s["pose6"], s["index"], coef)
    _, g2, _ = _gpu_grads(s["model"], x, s["pose6"], s["index"], coef)
    for k in WEIGHTS + ["code"]:
        assert torch.equal(g1[k], g2[k]), k
    rows = torch.nonzero(full1.abs().sum(-1)).reshape(-1).tolist()
    assert rows == [tt.GOLDEN_INDEX], rows


def test_m0_and_input_guards(setup):
    m = setup["model"]
    c = m.torso_individual_codes[setup["index"].cuda()]
    a, col, dx = m.forward_torso(torch.zeros(0, 2, device="cuda"), setup["pose6"].cuda(), c)
    (a.sum() + col.sum() + dx.sum()).backward()
    assert a.shape == (0, 1) and col.shape == (0, 3) and dx.shape == (0, 2)
    with pytest.raises(NotImplementedError):
        m.forward_torso(torch.zeros(4, 2, device="cuda", requires_grad=True), setup["pose6"].cuda(), c)
    with pytest.raises(NotImplementedError):
        m.forward_torso(torch.zeros(4, 2, device="cuda"), setup["pose6"].cuda().requires_grad_(True), c)
    with pytest.raises(ValueError):
        m.forward_torso(torch.zeros(4, 2, device="cuda"), setup["pose6"].cuda(), None)


def _golden_step_inputs(z):
    return {k: torch.from_numpy(z[f"b.{k}"]).cuda() for k in ("rays_o", "rays_d", "cond", "bg_coords", "bg_color", "gt")}


def test_torso_training_step_against_reference_golden_b(setup):
    """The reference's torso training step (render() in .train(), perturb=False, the task's loss, backward) restated on libgfpp's
    training ops and training-mode forward_torso, against tests/golden/train_torso.npz part (b)."""
    s = setup
    m = s["model"]
    z = np.load(GOLDEN)
    inp = _golden_step_inputs(z)
    m.zero_grad(set_to_none=True)
    res = tt.gfpp_train_step(m, inp["rays_o"], inp["rays_d"], inp["cond"], inp["bg_coords"], torch.from_numpy(z["pose6"]).cuda(),
                             s["index"].cuda(), inp["bg_color"], tt.GOLDEN_MAX_STEPS)
    tt.task_loss(res, inp["gt"], tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    torch.cuda.synchronize()
    for k in ("torso_alpha_map", "torso_rgb_map", "rgb_map", "weights_sum"):
        e = _rel(res[k].detach().reshape(-1), z[f"b.{k}"].reshape(-1))
        print(f"golden (b) {k}: rel {e:.2e}")
        assert e <= STEP_OUT, (k, e)
    params = dict(m.named_parameters())
    gg = {k: params[k].grad.cpu() for k in tt.TRAINABLE}
    gg["code"] = params["torso_individual_codes"].grad[tt.GOLDEN_INDEX].cpu()
    assert all(p.grad is None for k, p in params.items() if k not in tt.TRAINABLE + ["torso_individual_codes"]), "the head must stay frozen"
    _check_golden_grads(z, "b", gg)


def test_adam_steps_against_eager_restatement(setup):
    """The same step with the torso field in eager PyTorch (F.linear over train_ops.grid_encode with input gradients): the first
    step's gradients, then three Adam steps of both."""
    s = setup
    sc = s["sc"]
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = tt.GOLDEN_DS
    m.mlp_precision = "fp32"
    m = m.cuda().train()
    e = RADNeRFTorso(sc.hparams)
    e.load_state_dict(sc.state, strict=True)
    e.density_scale = tt.GOLDEN_DS
    e.mlp_precision = "fp32"
    e = e.cuda().train()
    P = {k: p for k, p in e.named_parameters() if k in tt.TRAINABLE}

    def eager_field(x, poses, c):
        return tt.eager_torso(e, P, x, poses, c, train_ops.grid_encode)

    z = np.load(GOLDEN)
    inp = _golden_step_inputs(z)
    pose6 = torch.from_numpy(z["pose6"]).cuda()
    idx = s["index"].cuda()
    names = tt.TRAINABLE + ["torso_individual_codes"]
    pa = [p for k, p in m.named_parameters() if k in names]
    pb = [p for k, p in e.named_parameters() if k in names]
    opt_a, opt_b = torch.optim.Adam(pa, lr=1e-3), torch.optim.Adam(pb, lr=1e-3)
    assert not torch.backends.cuda.matmul.allow_tf32    # the eager restatement is plain fp32
    la, lb = [], []
    for it in range(4):
        opt_a.zero_grad()
        opt_b.zero_grad()
        loss_a = tt.task_loss(tt.gfpp_train_step(m, inp["rays_o"], inp["rays_d"], inp["cond"], inp["bg_coords"], pose6, idx, inp["bg_color"],
                                                 tt.GOLDEN_MAX_STEPS), inp["gt"], tt.LAMBDA_WEIGHTS_ENTROPY)
        loss_b = tt.task_loss(tt.gfpp_train_step(e, inp["rays_o"], inp["rays_d"], inp["cond"], inp["bg_coords"], pose6, idx, inp["bg_color"],
                                                 tt.GOLDEN_MAX_STEPS, torso_field=eager_field), inp["gt"], tt.LAMBDA_WEIGHTS_ENTROPY)
        loss_a.backward()
        loss_b.backward()
        if it == 0:
            for k, a, b in zip(names, pa, pb):
                err = _rel(a.grad, b.grad)
                print(f"first-step gradient {k}: rel {err:.2e} against the eager restatement")
                assert err <= FIRST_STEP_REL, (k, err)
        la.append(loss_a.item())
        lb.append(loss_b.item())
        if it < 3:
            opt_a.step()
            opt_b.step()
    dl = max(abs(a - b) / abs(b) for a, b in zip(la, lb))
    dp = max((a.detach() - b.detach()).norm().item() / b.detach().norm().item() for a, b in zip(pa, pb))
    print(f"Adam x3: loss {la[0]:.6f} -> {la[-1]:.6f}; max rel loss diff {dl:.2e}; max rel L2 param diff {dp:.2e}")
    assert la[-1] < la[0]
    assert dl <= ADAM_LOSS_REL and dp <= ADAM_PARAM_REL, (dl, dp)
