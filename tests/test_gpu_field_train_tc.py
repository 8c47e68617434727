"""The tensor-core training field on the GPU (gfpp.h section J, RADNeRF.train_precision = "fp16").

  * forward against the rounding oracle (oracle/field_train_tc.py) and against libgfpp's fp32 field; training-mode and no_grad equal;
  * every gradient against the float64 oracle (cosine, relative L2) and against what it replaces: the eager restatement under fp16
    autocast must not be more than EAGER_FACTOR times closer to float64;
  * loss-scale independence: upstream gradients times 2^-20 and 2^12 give the same gradients times the scale; one GradScaler step;
  * determinism, M = 0 / 1 / ragged / several tiles per CTA, points outside the box;
  * render() in training mode against tests/golden/train_head.npz and 20 Adam steps beside the fp32 field;
  * train_precision = "fp32" is section G, bit for bit.

Each bar is at most about three times the value measured on an H100 (in its comment); each test prints what it measured.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF
from oracle import field_train as ft
from oracle import field_train_tc as ftc
from oracle import ops

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_head.npz")

FWD_ABS = 2e-5           # colour / ambient against the rounding oracle, absolute (measured 3.5e-6 to 7.4e-6)
FWD_SIGMA_REL = 1.5e-4   # sigma against the rounding oracle, relative to the largest sigma (measured 3.6e-5, 5.0e-5)
FWD_FP32_FACTOR = 8.0    # against libgfpp's fp32 field: this many times the two bars above (measured 3.3e-5 colour, 3.6e-4 sigma)
# Gradients against the float64 oracle.  The field amplifies operand rounding (tools/error_budget.py): an fp16-rounded activation
# moves the ambient coordinates across cells of the fine ambient-grid levels, where dy_dx jumps, and flips ReLUs at ties; the CPU
# rounding oracle shows the same errors (tests/test_oracle_field_train_tc.py), and fp16 autocast is 5 to 10 times further off.
# (The proposal for this arithmetic was cosine 0.999 and 2e-2 everywhere; only sigma_net.2, the colour net and the code reach it.)
GRAD_COS = 0.992         # cosine similarity: sigma and colour nets, ambient table, code (measured 0.99728 to 1.0)
GRAD_L2 = 0.15           # ... and relative L2 error (measured 5.6e-4 to 7.4e-2; per-level norms of the ambient table 4.5e-2)
GRAD_COS_UPSTREAM = 0.967  # what comes through the ambient grid's input gradient: ambient net, position table, cond (measured 0.98903 to 0.99659)
GRAD_L2_UPSTREAM = 0.4   # (measured 8.4e-2 to 1.48e-1; eager fp16 autocast on the same inputs: 0.73 to 1.19)
UPSTREAM = ("ambient_net.net.0.weight", "ambient_net.net.1.weight", "ambient_net.net.2.weight", "position_embedder.embeddings", "cond")
EAGER_FACTOR = 3.0       # relative L2 error against float64 <= this many times that of the eager field under fp16 autocast
                         # (measured: 0.02 to 0.14 times it -- the autocast field also rounds the tables and the inputs of tanh and exp)
SCALE_REL = 0.0          # weight / cond / code gradients under a scaled upstream gradient against scale * the unscaled ones: bit-equal
DET_TAB_REL = 5e-6       # table gradients, run to run (vector reductions in free order; measured 4.4e-8 to 1.5e-6)
RENDER_ABS = 3e-5        # rgb_map of the training render() against the reference golden (measured 8.7e-6)
ADAM_LOSS_REL = 3e-3     # 20 Adam steps: loss curve against the fp32 field's (measured 8.7e-4)

SHAPES = [(3, 4), (2, 0)]   # (ambient_coord_dim, individual_embedding_dim)


def _model(sc, hp, state, precision):
    m = RADNeRF(hp)
    m.load_state_dict(state, strict=True)
    m.density_scale = sc.density_scale
    m.train_precision = precision
    return m.cuda()


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
    model = _model(sc, hp, state, "fp16")
    g = torch.Generator().manual_seed(7)
    M = 3001                                         # not a multiple of the tile
    lo, hi = model.aabb_train[:3].cpu(), model.aabb_train[3:].cpu()
    xyzs = lo + (hi - lo) * torch.rand(M, 3, generator=g)
    dirs = F.normalize(torch.randn(M, 3, generator=g), dim=-1)
    cond_feat = model.cal_cond_feat(scn.cond_window(sc.cond, 1, sc.hparams["smo_win_size"]).cuda()).detach().reshape(1, -1)
    code = state["individual_embeddings"][2].clone() if ind_dim else None
    gs, gc, ga = torch.randn(M, generator=g), torch.randn(M, 3, generator=g), torch.randn(M, amb_dim, generator=g)
    return dict(sc=sc, hp=hp, state=state, model=model, xyzs=xyzs, dirs=dirs, cond=cond_feat.cpu(), code=code, gs=gs, gc=gc, ga=ga)


def _loss(out, s, M, scale=1.0, dev="cuda"):
    sig, col, amb = out
    gs, gc, ga = (s[k][:M].to(dev) * scale for k in ("gs", "gc", "ga"))
    return (sig * gs.to(sig.dtype)).sum() + (col * gc.to(sig.dtype)).sum() + (amb * ga.to(sig.dtype)).sum()


def _gpu_field(s, M=None, scale=1.0, model=None, xyzs=None):
    """libgfpp's forward + backward through RADNeRF.forward; returns outputs and the gradients by name."""
    m = s["model"] if model is None else model
    m.zero_grad(set_to_none=True)
    x = s["xyzs"] if xyzs is None else xyzs
    M = x.shape[0] if M is None else M
    cond = s["cond"].cuda().requires_grad_(True)
    code = s["code"].cuda().requires_grad_(True) if s["code"] is not None else None
    out = m.forward(x[:M].cuda(), s["dirs"][:M].cuda(), cond, code)
    _loss(out, s, M, scale).backward()
    grads = {k: p.grad.detach().cpu().clone() for k, p in m.named_parameters() if k in ft.TRAINABLE}
    grads["cond"] = cond.grad.cpu()
    if code is not None:
        grads["code"] = code.grad.cpu()
    torch.cuda.synchronize()
    return tuple(o.detach().cpu() for o in out), grads


def _oracle_field(s, fwd, dtype=torch.float32):
    p = ft.field_params(s["state"], dtype)
    cond = s["cond"].clone().to(dtype).requires_grad_(True)
    code = s["code"].clone().to(dtype).requires_grad_(True) if s["code"] is not None else None
    out = fwd(p, s["hp"], s["xyzs"], s["dirs"].to(dtype), cond, code)
    _loss(out, s, s["xyzs"].shape[0], dev="cpu").backward()
    grads = {k: p[k].grad for k in ft.TRAINABLE}
    grads["cond"] = cond.grad
    if code is not None:
        grads["code"] = code.grad
    return tuple(o.detach() for o in out), grads


def _autocast_field(s):
    """The eager restatement under fp16 autocast, the arithmetic of the reference's amp: true."""
    m = s["model"]
    P = {k: s["state"][k].detach().clone().cuda().requires_grad_(True) for k in ft.TRAINABLE}
    cond = s["cond"].cuda().requires_grad_(True)
    code = s["code"].cuda().requires_grad_(True) if s["code"] is not None else None
    with torch.autocast("cuda", dtype=torch.float16):
        out = ft.eager_field(m, P, s["xyzs"].cuda(), s["dirs"].cuda(), cond, code, train_ops.grid_encode)
    _loss(tuple(o.float() for o in out), s, s["xyzs"].shape[0]).backward()
    grads = {k: P[k].grad.float().cpu() for k in ft.TRAINABLE}
    grads["cond"] = cond.grad.float().cpu()
    if code is not None:
        grads["code"] = code.grad.float().cpu()
    return grads


def _l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _cos(a, b):
    return F.cosine_similarity(a.double().reshape(1, -1), b.double().reshape(1, -1)).item()


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _level_norms(model, name, g):
    off = getattr(model, name.split(".")[0]).offsets.cpu().tolist()
    return torch.tensor([float(g[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)], dtype=torch.float64)


def test_forward_against_rounding_oracle_and_fp32_field(setup):
    s = setup
    m = s["model"]
    (sig, col, amb), _ = _gpu_field(s)
    (rs, rc, ra), _ = _oracle_field(s, ftc.field_forward)
    m32 = _model(s["sc"], s["hp"], s["state"], "fp32")
    (fs, fc, fa), _ = _gpu_field(s, model=m32)
    for name, (os_, oc, oa), k in (("rounding oracle", (rs, rc, ra), 1.0), ("fp32 field", (fs, fc, fa), FWD_FP32_FACTOR)):
        e = [(sig - os_).abs().max().item() / os_.abs().max().item(), (col - oc).abs().max().item(), (amb - oa).abs().max().item()]
        print(f"forward vs {name}: sigma rel {e[0]:.2e}, colour abs {e[1]:.2e}, ambient abs {e[2]:.2e}")
        assert e[0] <= k * FWD_SIGMA_REL and e[1] <= k * FWD_ABS and e[2] <= k * FWD_ABS, (name, e)
    with torch.no_grad():
        out = m.forward(s["xyzs"].cuda(), s["dirs"].cuda(), s["cond"].cuda(), s["code"].cuda() if s["code"] is not None else None)
    assert torch.equal(out[0].cpu(), sig) and torch.equal(out[1].cpu(), col) and torch.equal(out[2].cpu(), amb)
    assert all(o.dtype == torch.float32 for o in out)
    with torch.autocast("cuda", dtype=torch.float16), torch.no_grad():
        out = m.forward(s["xyzs"].cuda(), s["dirs"].cuda(), s["cond"].cuda(), s["code"].cuda() if s["code"] is not None else None)
    assert out[0].dtype == torch.float32 and torch.equal(out[1].cpu(), col)


def test_gradients_against_float64_and_autocast(setup):
    s = setup
    _, g = _gpu_field(s)
    _, r64 = _oracle_field(s, ft.field_forward, torch.float64)
    ac = _autocast_field(s)
    bad = []
    for k in r64:
        cos, l2, l2_ac = _cos(g[k], r64[k]), _l2(g[k], r64[k]), _l2(ac[k], r64[k])
        print(f"grad {k}: cosine {cos:.6f}, rel L2 {l2:.2e} (eager fp16 autocast {l2_ac:.2e})")
        up = k in UPSTREAM
        if cos < (GRAD_COS_UPSTREAM if up else GRAD_COS) or l2 > (GRAD_L2_UPSTREAM if up else GRAD_L2):
            bad.append((k, cos, l2))
        if np.isfinite(l2_ac) and l2 > EAGER_FACTOR * l2_ac:
            bad.append((k, l2, l2_ac))
        if k.endswith("embeddings"):
            en = _rel(_level_norms(s["model"], k, g[k]), _level_norms(s["model"], k, r64[k]))
            print(f"grad {k}: per-level norms rel {en:.2e}")
            if en > (GRAD_L2_UPSTREAM if up else GRAD_L2):
                bad.append((k, "level norms", en))
    assert not bad, bad


def test_loss_scale_independence(setup):
    s = setup
    _, g1 = _gpu_field(s)
    for scale in (2.0 ** -20, 2.0 ** 12):
        _, gk = _gpu_field(s, scale=scale)
        for k in g1:
            assert torch.isfinite(gk[k]).all(), k
            tab = k.endswith("embeddings")   # scattered in free order: equal up to DET_TAB_REL
            e = _rel(gk[k], g1[k] * scale)
            print(f"scale {scale:.1e} grad {k}: rel {e:.2e}")
            assert e <= (DET_TAB_REL if tab else SCALE_REL), (k, scale, e)


def test_grad_scaler_step(setup):
    s = setup
    m = _model(s["sc"], s["hp"], s["state"], "fp16")
    before = m.sigma_net.net[1].weight.detach().clone()
    opt = torch.optim.Adam([p for k, p in m.named_parameters() if k in ft.TRAINABLE], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    code = s["code"].cuda() if s["code"] is not None else None
    with torch.autocast("cuda", dtype=torch.float16):
        out = m.forward(s["xyzs"].cuda(), s["dirs"].cuda(), s["cond"].cuda(), code)
        loss = _loss(out, s, s["xyzs"].shape[0]) / s["xyzs"].shape[0]
    scaler.scale(loss).backward()
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == 2.0 ** 16, "the step was skipped: a gradient was not finite"
    assert (m.sigma_net.net[1].weight.detach() - before).abs().max().item() > 0


@pytest.mark.parametrize("value", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("which", ["gc", "gs"], ids=["grad_color", "grad_sigma"])
def test_non_finite_upstream_skips_the_step(setup, which, value):
    """One inf or NaN in the upstream gradient: a weight gradient comes out non-finite and a GradScaler step is skipped (loss scaling
    relies on it; block_scale's fmaxf leaves a NaN out of the block's largest magnitude, so it must travel through the products)."""
    s = setup
    bad = dict(s)
    bad[which] = s[which].clone()
    bad[which].view(-1)[1234] = value
    m = _model(s["sc"], s["hp"], s["state"], "fp16")
    before = {k: p.detach().clone() for k, p in m.named_parameters() if k in ft.TRAINABLE}
    opt = torch.optim.Adam([p for k, p in m.named_parameters() if k in ft.TRAINABLE], lr=1e-3)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    code = s["code"].cuda() if s["code"] is not None else None
    out = m.forward(s["xyzs"].cuda(), s["dirs"].cuda(), s["cond"].cuda(), code)
    scaler.scale(_loss(out, bad, s["xyzs"].shape[0])).backward()
    finite = {k: bool(torch.isfinite(p.grad).all()) for k, p in m.named_parameters() if k in ft.TRAINABLE}
    scaler.step(opt)
    scaler.update()
    print(f"{which}[1234] = {value}: non-finite gradients {[k for k, v in finite.items() if not v]}; scale {scaler.get_scale():.0f}")
    assert not all(finite[k] for k in ft.TRAINABLE[:8]), finite
    assert scaler.get_scale() < 2.0 ** 16, "the step was not skipped"
    assert all(torch.equal(p.detach(), before[k]) for k, p in m.named_parameters() if k in ft.TRAINABLE)


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


def test_edges(setup):
    s = setup
    A = s["model"].ambient_coord_dim
    (sig, col, amb), g = _gpu_field(s, M=0)
    assert sig.shape == (0,) and col.shape == (0, 3) and amb.shape == (0, A)
    assert all(float(v.abs().max()) == 0.0 for v in g.values() if v.numel())
    (sall, call, aall), _ = _gpu_field(s)
    for M in (1, 130):
        (sm, cm, am), gm = _gpu_field(s, M=M)
        assert torch.equal(sm, sall[:M]) and torch.equal(cm, call[:M]) and torch.equal(am, aall[:M])
        assert all(torch.isfinite(v).all() for v in gm.values())
    # several tiles per CTA: the same 3001 points repeated; the weight gradients are the sums, so `reps` times the single batch's
    reps = 132 * 128 * 3 // 3001 + 2
    big = dict(s)
    for k in ("xyzs", "dirs", "gs", "gc", "ga"):
        big[k] = s[k].repeat(reps, *([1] * (s[k].dim() - 1)))
    (sb, cb, ab), gb = _gpu_field(big)
    assert torch.equal(sb[-3001:], sall) and torch.equal(cb[:3001], call)
    _, g1 = _gpu_field(s)
    for k in g1:
        e = _l2(gb[k], g1[k] * reps)
        print(f"{reps} x 3001 points, grad {k}: rel L2 {e:.2e} against {reps} x the single batch")
        assert e <= GRAD_L2, (k, e)
    # points outside the box: zero features, no table gradient
    far = s["xyzs"][:200] * 0 + 10.0
    for t in ("position_embedder.embeddings",):
        _, gf = _gpu_field(s, M=200, xyzs=far)
        assert float(gf[t].abs().max()) == 0.0
        assert all(torch.isfinite(v).all() for v in gf.values())


def _train_model(precision):
    sc = scn.Scene(H=32, W=32, T=4, torso=False, density_scale=8.0)
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m.train_precision = precision
    return m.cuda().train()


def test_training_render_and_adam_steps():
    ops.build()
    G = np.load(GOLDEN)

    def t(k):
        return torch.from_numpy(G[k]).cuda()

    curves = {}
    for precision in ("fp32", "fp16"):
        m = _train_model(precision)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        target = t("bg_color").reshape(-1, 3).flip(0)
        losses = []
        for it in range(20):
            opt.zero_grad()
            res = m.render(t("rays_o"), t("rays_d"), t("cond"), None, None, index=2, bg_color=t("bg_color"), perturb=False, max_steps=16)
            if it == 0 and precision == "fp16":
                assert torch.equal(res["position"].cpu(), torch.from_numpy(G["position"])), "samples differ from the reference's"
                e = (res["rgb_map"].detach().cpu().reshape(G["rgb_map"].shape) - torch.from_numpy(G["rgb_map"])).abs().max().item()
                print(f"training render rgb_map vs the reference golden: max abs {e:.2e}")
                assert e <= RENDER_ABS
            loss = ((res["rgb_map"].reshape(-1, 3) - target) ** 2).mean() + 1e-3 * res["ambient"].mean()
            loss.backward()
            opt.step()
            losses.append(loss.item())
        curves[precision] = losses
    d = max(abs(a - b) / abs(b) for a, b in zip(curves["fp16"], curves["fp32"]))
    print(f"Adam x20: fp16 loss {curves['fp16'][0]:.6f} -> {curves['fp16'][-1]:.6f}, fp32 {curves['fp32'][0]:.6f} -> {curves['fp32'][-1]:.6f}; "
          f"max rel diff {d:.2e}")
    assert curves["fp16"][-1] < curves["fp16"][0]
    assert d <= ADAM_LOSS_REL, d


def test_fp32_precision_is_section_g(setup):
    """train_precision = "fp32" (the default) runs gfpp_field_forward / gfpp_field_backward: bit-identical to calling them directly."""
    s = setup
    m = _model(s["sc"], s["hp"], s["state"], "fp32")
    assert RADNeRF(s["hp"]).train_precision == "fp32"
    (sig, col, amb), g = _gpu_field(s, model=m)
    L, dev = _capi.lib(), torch.device("cuda")
    M, A = s["xyzs"].shape[0], m.ambient_coord_dim
    x, dr, c = s["xyzs"].cuda(), s["dirs"].cuda(), s["cond"].cuda().reshape(-1)
    cd = s["code"].cuda() if s["code"] is not None else None
    keep = []
    d = train_ops._field_desc(m, cd, keep)
    ws = torch.empty(L.gfpp_field_backward_workspace_bytes(M), dtype=torch.uint8, device=dev)
    o = [torch.empty(M, device=dev), torch.empty(M, 3, device=dev), torch.empty(M, A, device=dev)]
    _capi.check(L.gfpp_field_forward(ctypes.byref(d), x.data_ptr(), dr.data_ptr(), M, c.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(),
                                     ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_field_forward")
    assert torch.equal(o[0].cpu(), sig) and torch.equal(o[1].cpu(), col) and torch.equal(o[2].cpu(), amb)
    params = [dict(m.named_parameters())[k] for k in ft.TRAINABLE]
    gw = [torch.empty_like(p) for p in params[:8]]
    gt = [torch.zeros_like(p) for p in params[8:]]
    g_cond = torch.empty(64, device=dev)
    g_code = torch.empty_like(cd) if cd is not None else None
    ptrs = (ctypes.c_void_p * 8)(*[t.data_ptr() for t in gw])
    up = [s[k].cuda().contiguous() for k in ("gs", "gc", "ga")]
    _capi.check(L.gfpp_field_backward(ctypes.byref(d), x.data_ptr(), dr.data_ptr(), M, c.data_ptr(), up[0].data_ptr(), up[1].data_ptr(), up[2].data_ptr(),
                                      ctypes.byref(ptrs), g_cond.data_ptr(), None if g_code is None else g_code.data_ptr(), gt[0].data_ptr(),
                                      gt[1].data_ptr(), ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_field_backward")
    for k, t in zip(ft.TRAINABLE[:8], gw):
        assert torch.equal(t.cpu(), g[k]), k
    assert torch.equal(g_cond.cpu(), g["cond"].reshape(-1))
    if g_code is not None:
        assert torch.equal(g_code.cpu(), g["code"])
    for k, t in zip(ft.TRAINABLE[8:], gt):
        assert _rel(t.cpu(), g[k]) <= DET_TAB_REL, k
