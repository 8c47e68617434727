"""The trainable head field on the GPU (gfpp.h section G, RADNeRF.forward, the training branch of RADNeRF.render).

  * forward against the CPU oracle (oracle/field_train.py) and raw sigma against density() of an fp32 model;
  * every gradient (eight weights, cond_feat, individual code, both tables) against the oracle under autograd;
  * determinism: two backward runs are bit-identical except the table gradients (vector reductions in free order);
  * M = 0 and M not a multiple of the 64-point tile;
    these four for the May shapes (ambient_coord_dim 3, ind_dim 4) and for a 2-D ambient grid without individual codes;
  * the training render() + backward against tests/golden/train_head.npz: the reference's own RADNeRF.render and .backward;
  * the first step's gradients and 20 Adam steps with libgfpp against an eager fp32 restatement over train_ops, then an eval render
    of the trained model against a freshly constructed one loaded with its state_dict.

Bounds are about twice the values measured on an H100 (DESIGN.md section 3); each test prints what it measured.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF
from oracle import field_train as ft
from oracle import ops

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_head.npz")

# bounds: about twice the values measured on an H100 (DESIGN.md section 3), on the scene's default state.  (With
# tests/helpers.lively_state the field is so ill-conditioned that the fp32 oracle itself is ~3e-2 from a float64 evaluation.)
FWD_REL = 1e-5          # sigma / colour / ambient, relative to the largest |value| (measured 3.9e-6)
GRAD_REL = 1e-4         # gradients at random points with random upstream gradients, relative to the largest |entry| (measured <= 3.5e-5)
REF_ROUNDING_FACTOR = 3.0
FLIP_BAND = 1e-4        # points with a ReLU pre-activation this close to 0 (relative to the layer's largest) get no upstream gradient:
                        # the kernel sums in another order than the oracle (and folds the conditioning / code columns into biases), so
                        # a ReLU at such a tie may flip, which moves a whole row of a weight gradient by a gradient-sized amount
GOLDEN_TIE = {"grad.color_net.net.0.weight": 2e-3, "grad.individual_code": 1e-3}
GOLDEN_COND_TIE = 5e-3   # measured <= 2.7e-3
GOLDEN_TABLE_REL = 1e-3  # table gradients against the reference's fp32 ones (measured 2.8e-4): they come through the ambient-net gradients,
                         # which the reference itself computes up to 9e-4 off float64 (column sums that cancel)
GOLDEN_NORM_REL = 5e-3   # per-level norms of the table gradients (measured 2.0e-3 on the ambient table: the colour-net tie of GOLDEN_TIE
                         # reaches every ambient-table entry its sample touches)   # the golden's samples cannot be filtered: a colour-net ReLU tie flips there (8.0e-4
                        # from the float64 gradient, the reference 1.7e-6), driven by the summation order and the 1-ulp difference of
                        # cal_cond_feat between the GPU and the reference's CPU
GOLDEN_REL = 5e-5       # the training render() and its gradients against the reference golden
DET_TAB_REL = 5e-6      # table gradients, run to run (measured 5.6e-8 to 2.3e-6)
FIRST_STEP_REL = 1e-3   # first-step gradients, libgfpp against the eager restatement
ADAM_LOSS_REL = 3e-3    # 20 Adam steps: loss curves (measured 2.5e-4 to 1.25e-3 over four runs: the eager leg's table scatter order varies)
ADAM_PARAM_REL = 0.2    # 20 Adam steps: parameters, relative L2 (measured 9.7e-2: Adam turns noise-level gradients into full steps)

SHAPES = [(3, 4), (2, 0)]   # (ambient_coord_dim, individual_embedding_dim)


@pytest.fixture(scope="module", params=SHAPES, ids=lambda v: f"amb{v[0]}_ind{v[1]}")
def setup(request):
    amb_dim, ind_dim = request.param
    ops.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    sc = scn.Scene(H=32, W=32, T=4, torso=False, density_scale=8.0)
    hp = may_hparams(max_steps=16, ambient_coord_dim=amb_dim, individual_embedding_dim=ind_dim)
    state = sc.state if (amb_dim, ind_dim) == (3, 4) else scn.make_state(torso=False, hparams=hp)
    if ind_dim == 0:
        state = {k: v for k, v in state.items() if k != "individual_embeddings"}
    model = RADNeRF(hp)
    model.load_state_dict(state, strict=True)
    model.density_scale = sc.density_scale
    model = model.cuda()
    g = torch.Generator().manual_seed(7)
    M = 3001                                         # not a multiple of the tile
    lo = model.aabb_train[:3].cpu()
    hi = model.aabb_train[3:].cpu()
    xyzs = lo + (hi - lo) * torch.rand(M, 3, generator=g)
    dirs = F.normalize(torch.randn(M, 3, generator=g), dim=-1)
    cond_feat = model.cal_cond_feat(scn.cond_window(sc.cond, 1, sc.hparams["smo_win_size"]).cuda()).detach().reshape(1, -1)
    code = state["individual_embeddings"][2].clone() if ind_dim else None
    gs = torch.randn(M, generator=g)
    gc = torch.randn(M, 3, generator=g)
    ga = torch.randn(M, amb_dim, generator=g)
    # points at a ReLU tie of the colour net's first layer (FLIP_BAND) carry no upstream gradient
    trace = {}
    ft.field_forward(ft.field_params(state), hp, xyzs, dirs, cond_feat.cpu(), code, trace=trace)
    tie = torch.zeros(M, dtype=torch.bool)
    for pre in trace["relu_pre"]:
        tie |= (pre.abs() < FLIP_BAND * pre.abs().max()).any(1)
    gs[tie], gc[tie], ga[tie] = 0, 0, 0
    print(f"[amb {amb_dim}, ind {ind_dim}] {int(tie.sum())} of {M} points at a ReLU tie")
    return dict(sc=sc, hp=hp, state=state, model=model, xyzs=xyzs, dirs=dirs, cond=cond_feat.cpu(), code=code, gs=gs, gc=gc, ga=ga)


def _gpu_field(s, M=None):
    """libgfpp's forward + backward through RADNeRF.forward; returns outputs and the gradients by name."""
    m = s["model"]
    m.zero_grad(set_to_none=True)
    M = s["xyzs"].shape[0] if M is None else M
    cond = s["cond"].cuda().requires_grad_(True)
    code = s["code"].cuda().requires_grad_(True) if s["code"] is not None else None
    sig, col, amb = m.forward(s["xyzs"][:M].cuda(), s["dirs"][:M].cuda(), cond, code)
    loss = (sig * s["gs"][:M].cuda()).sum() + (col * s["gc"][:M].cuda()).sum() + (amb * s["ga"][:M].cuda()).sum()
    loss.backward()
    grads = {k: p.grad.detach().cpu().clone() for k, p in m.named_parameters() if k in ft.TRAINABLE}
    grads["cond"] = cond.grad.cpu()
    if code is not None:
        grads["code"] = code.grad.cpu()
    torch.cuda.synchronize()
    return (sig.detach().cpu(), col.detach().cpu(), amb.detach().cpu()), grads


def _oracle_field(s, dtype=torch.float32):
    p = ft.field_params(s["state"], dtype)
    cond = s["cond"].clone().to(dtype).requires_grad_(True)
    code = s["code"].clone().to(dtype).requires_grad_(True) if s["code"] is not None else None
    sig, col, amb = ft.field_forward(p, s["hp"], s["xyzs"], s["dirs"].to(dtype), cond, code)
    loss = (sig * s["gs"].to(dtype)).sum() + (col * s["gc"].to(dtype)).sum() + (amb * s["ga"].to(dtype)).sum()
    loss.backward()
    grads = {k: p[k].grad for k in ft.TRAINABLE}
    grads["cond"] = cond.grad
    if code is not None:
        grads["code"] = code.grad
    return (sig.detach(), col.detach(), amb.detach()), grads


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def test_forward_against_oracle_and_density(setup):
    s = setup
    (sig, col, amb), _ = _gpu_field(s)
    (rs, rc, ra), _ = _oracle_field(s)
    e = [_rel(sig, rs), _rel(col, rc), _rel(amb, ra)]
    print(f"forward rel err sigma {e[0]:.2e} colour {e[1]:.2e} ambient {e[2]:.2e}")
    assert max(e) <= FWD_REL, e
    m = s["model"]
    with torch.no_grad():
        d = m.density(s["xyzs"].cuda(), s["cond"].cuda())["sigma"].cpu()
    ed = _rel(sig, d)
    print(f"raw sigma vs density() of the fp32 model: rel {ed:.2e}")
    assert ed <= FWD_REL


def test_gradients_against_oracle(setup):
    """Against the fp32 oracle within GRAD_REL, or -- where a gradient is a column sum that cancels, so that any fp32 evaluation
    order is visibly rounded -- no further from the oracle with float64 dense layers than REF_ROUNDING_FACTOR times the fp32 oracle is."""
    s = setup
    _, g = _gpu_field(s)
    _, r = _oracle_field(s)
    _, r64 = _oracle_field(s, torch.float64)
    for k in r:
        e = _rel(g[k], r[k])
        e_gpu, e_orc = _rel(g[k].double(), r64[k].double()), _rel(r[k].double(), r64[k].double())
        print(f"grad {k}: rel {e:.2e}; to float64: libgfpp {e_gpu:.2e}, fp32 oracle {e_orc:.2e}")
        assert e <= GRAD_REL or e_gpu <= REF_ROUNDING_FACTOR * e_orc, (k, e, e_gpu, e_orc)


def test_backward_is_deterministic(setup):
    s = setup
    out1, g1 = _gpu_field(s)
    out2, g2 = _gpu_field(s)
    for a, b in zip(out1, out2):
        assert torch.equal(a, b)
    for k in g1:
        if k.endswith("embeddings"):
            d = _rel(g1[k], g2[k])
            print(f"table gradient {k}: run-to-run rel {d:.2e}")
            assert d <= DET_TAB_REL, (k, d)
        else:
            assert torch.equal(g1[k], g2[k]), k


def test_m0_and_ragged_m(setup):
    s = setup
    (sig, col, amb), g = _gpu_field(s, M=0)
    assert sig.shape == (0,) and col.shape == (0, 3) and amb.shape == (0, s["model"].ambient_coord_dim)
    assert all(float(v.abs().max()) == 0.0 for v in g.values() if v.numel())
    (s130, c130, a130), _ = _gpu_field(s, M=130)
    (sall, call, aall), _ = _gpu_field(s)
    assert torch.equal(s130, sall[:130]) and torch.equal(c130, call[:130]) and torch.equal(a130, aall[:130])


def test_training_render_against_reference_golden():
    """model.train(); render() + backward on the inputs of tests/golden/train_head.npz (the reference's own RADNeRF.render in training
    mode and its backward, oracle/make_train_golden.py): outputs, samples and every gradient, the conditioning nets' included."""
    ops.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    G = np.load(GOLDEN)
    sc = scn.Scene(H=32, W=32, T=4, torso=False, density_scale=8.0)
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m = m.cuda().train()

    def t(k):
        return torch.from_numpy(G[k]).cuda()

    res = m.render(t("rays_o"), t("rays_d"), t("cond"), None, None, index=2, bg_color=t("bg_color"), perturb=False, max_steps=16)
    loss = (res["rgb_map"].reshape(-1, 3) * t("coef_rgb")).sum() + (res["weights_sum"] * t("coef_ws")).sum() + (res["ambient"] * t("coef_amb")).sum()
    loss.backward()
    m.eval()
    assert m.local_step == 1
    assert set(res) >= {"weights_sum", "ambient", "position", "depth_map", "rgb_map"}
    assert torch.equal(res["position"].cpu(), torch.from_numpy(G["position"])), "samples differ from the reference's"
    params = dict(m.named_parameters())
    checks = [(k, res[k].detach()) for k in ("rgb_map", "weights_sum", "ambient", "depth_map")]
    checks += [("grad." + k, params[k].grad) for k in ft.TRAINABLE[:8]]
    checks += [("grad.individual_code", params["individual_embeddings"].grad[2])]
    checks += [(k, params[k[5:]].grad) for k in G.files if k.startswith(("grad.cond_prenet.", "grad.cond_att_net."))]
    for k, got in checks:
        got = got.cpu().reshape(G[k].shape)
        e = _rel(got, torch.from_numpy(G[k]))
        k64 = k.replace("grad.", "grad64.")
        if k64 in G.files:
            # where a weight gradient is a column sum that cancels, the reference's own fp32 result is off the float64 one by up to
            # 1.7e-2: libgfpp must be no further from float64 than REF_ROUNDING_FACTOR times the reference is (or within GOLDEN_REL)
            exact = torch.from_numpy(G[k64]).double()
            e_gpu, e_ref = _rel(got.double(), exact), _rel(torch.from_numpy(G[k]).double(), exact)
            print(f"golden {k}: rel {e:.2e}; to float64: libgfpp {e_gpu:.2e}, reference {e_ref:.2e}")
            assert e <= GOLDEN_TIE.get(k, GOLDEN_REL) or e_gpu <= REF_ROUNDING_FACTOR * e_ref, (k, e, e_gpu, e_ref)
        else:
            print(f"golden {k}: rel {e:.2e}")
            # the conditioning nets' gradients come through grad_cond, downstream of the same colour-net tie (GOLDEN_TIE)
            assert e <= (GOLDEN_COND_TIE if k.startswith("grad.cond_") else GOLDEN_REL), (k, e)
    for tname in ("position_embedder", "ambient_embedder"):
        gr = params[f"{tname}.embeddings"].grad.cpu()
        e = _rel(gr[torch.from_numpy(G[f"{tname}.sample_idx"])], torch.from_numpy(G[f"{tname}.sample_grad"]))
        off = getattr(m, tname).offsets.cpu().tolist()
        norms = torch.tensor([float(gr[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)], dtype=torch.float64)
        en = _rel(norms, torch.from_numpy(G[f"{tname}.level_norms"]))
        print(f"golden {tname} table gradient: sampled entries rel {e:.2e}, per-level norms rel {en:.2e}")
        assert e <= GOLDEN_TABLE_REL and en <= GOLDEN_NORM_REL, (tname, e, en)
    assert float(params["individual_embeddings"].grad[[0, 1, 3]].abs().max()) == 0.0


def _eager_field(m, P, xyzs, dirs, cond_feat, code):
    return ft.eager_field(m, P, xyzs, dirs, cond_feat, code, train_ops.grid_encode)


def test_adam_steps_against_eager_restatement(setup):
    """The first step's gradients against the eager restatement: the check of gradient scale and of small errors.  Adam is invariant
    to a constant scale on the gradient and turns noise-level differences into full steps, so the 20 steps after it only show that
    training tracks the eager path; the per-gradient oracle and golden tests carry the accuracy."""
    s = setup
    sc = s["sc"]
    if s["code"] is None:
        pytest.skip("the training loop runs on the May shapes")
    m = RADNeRF(sc.hparams)
    m.load_state_dict(s["state"], strict=True)
    m.density_scale = sc.density_scale
    m = m.cuda()
    P = {k: s["state"][k].detach().clone().cuda().requires_grad_(True) for k in ft.TRAINABLE + ["individual_embeddings"]}
    fi = sc.frame_inputs(2)
    rays_o, rays_d = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
    nears, fars = train_ops.near_far_from_aabb(rays_o, rays_d, m.aabb_train, m.min_near)
    xyzs, dirs, deltas, rays = train_ops.march_rays_train(rays_o, rays_d, m.bound, m.density_bitfield, m.cascade, m.grid_size, nears, fars,
                                                          None, 0, False, 128, False, 0, sc.hparams["max_steps"])
    with torch.no_grad():
        cond_feat = m.cal_cond_feat(fi["cond"].cuda()).reshape(1, -1)
    target = fi["bg_color"].cuda().reshape(-1, 3).flip(0)
    mine = [p for k, p in m.named_parameters() if k in P]
    names = [k for k, p in m.named_parameters() if k in P]
    opt_a = torch.optim.Adam(mine, lr=1e-3)
    opt_b = torch.optim.Adam([P[k] for k in names], lr=1e-3)

    def step(field, params_code):
        sig, col, amb = field
        ws, asum, _, image = train_ops.composite_rays_train(sig * m.density_scale, col, amb.abs().sum(-1), deltas, rays)
        img = image + (1 - ws).unsqueeze(-1)
        return ((img - target) ** 2).mean() + 1e-3 * asum.mean()

    opt_a.zero_grad()
    step(m.forward(xyzs, dirs, cond_feat, m.individual_embeddings[1]), None).backward()
    opt_b.zero_grad()
    step(_eager_field(m, P, xyzs, dirs, cond_feat, P["individual_embeddings"][1]), None).backward()
    for k, p in zip(names, mine):
        e = _rel(p.grad, P[k].grad) if k != "individual_embeddings" else _rel(p.grad[1], P[k].grad[1])
        print(f"first-step gradient {k}: rel {e:.2e} against the eager restatement")
        assert e <= FIRST_STEP_REL, (k, e)

    la, lb = [], []
    for it in range(20):
        opt_a.zero_grad()
        loss_a = step(m.forward(xyzs, dirs, cond_feat, m.individual_embeddings[1]), None)
        loss_a.backward()
        opt_a.step()
        opt_b.zero_grad()
        loss_b = step(_eager_field(m, P, xyzs, dirs, cond_feat, P["individual_embeddings"][1]), None)
        loss_b.backward()
        opt_b.step()
        la.append(loss_a.item())
        lb.append(loss_b.item())
    dl = max(abs(a - b) / abs(b) for a, b in zip(la, lb))
    dp = max((p.detach() - P[k].detach()).norm().item() / P[k].detach().norm().item() for k, p in zip(names, mine))
    dmove = min((p.detach() - s["state"][k].cuda()).abs().max().item() for k, p in zip(names, mine) if k != "individual_embeddings")
    print(f"Adam x20: loss {la[0]:.6f} -> {la[-1]:.6f}; max rel loss diff {dl:.2e}; max rel L2 param diff {dp:.2e}; min param move {dmove:.2e}")
    assert la[-1] < la[0]
    assert dl <= ADAM_LOSS_REL and dp <= ADAM_PARAM_REL, (dl, dp)

    # an eval render of the trained model equals that of a fresh model loaded with its state_dict
    m.eval()
    fresh = RADNeRF(sc.hparams)
    fresh.load_state_dict(m.state_dict(), strict=True)
    fresh.density_scale = m.density_scale
    fresh = fresh.cuda().eval()
    args = (fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda())
    a = m.render(*args, bg_color=fi["bg_color"].cuda(), T_thresh=sc.T_thresh, max_steps=sc.hparams["max_steps"])["rgb_map"]
    b = fresh.render(*args, bg_color=fi["bg_color"].cuda(), T_thresh=sc.T_thresh, max_steps=sc.hparams["max_steps"])["rgb_map"]
    m0 = RADNeRF(sc.hparams)
    m0.load_state_dict(s["state"], strict=True)
    m0.density_scale = m.density_scale
    c = m0.cuda().eval().render(*args, bg_color=fi["bg_color"].cuda(), T_thresh=sc.T_thresh, max_steps=sc.hparams["max_steps"])["rgb_map"]
    assert torch.equal(a, b)
    assert (a - c).abs().max().item() > 0, "the eval render must use the trained weights"


def test_wrong_sized_conditioning_raises(setup):
    s = setup
    m = s["model"]
    x, d = s["xyzs"][:8].cuda(), s["dirs"][:8].cuda()
    code = s["code"].cuda() if s["code"] is not None else None
    with pytest.raises(ValueError, match="cond_feat"):
        m.forward(x, d, s["cond"].cuda().repeat(2, 1), code)
    if code is not None:
        with pytest.raises(ValueError, match="individual_code"):
            m.forward(x, d, s["cond"].cuda(), code[:2])
