"""The tensor-core training field (gfpp.h section J, RADNeRF.train_precision = "fp16") against its own rounding model,
oracle/field_train_tc.py, at training-step scale (a step of the May configs marches 65 536 rays into a few hundred thousand samples):

  * outputs and every gradient at M = 3 001, 16 896 (132 CTAs x one 128-point tile), 16 897 (one CTA owns two tiles, the last holds
    one point), 65 537 and 262 144;
  * one call whose tiles alternate between upstream gradients at 2^12 and at 2^-40: the per-tile block scale keeps the faint tiles'
    bits, down to the position-table entries only they reach;
  * determinism at 262 144 points, and a grid-stride forward that is pointwise;
  * the steady-state training step in fp16: render() after update_extra_state has set mean_count, where M is below the sample count.

The oracle rounds exactly the operands the kernels round, with the kernels' power of two per 128-point block (block_scale); what is
left is the order of the fp32 sums inside wgmma and the rare one-ulp fp16 operand flip that follows from it.  Two kinds of points get
no upstream gradient, as in tests/test_gpu_train_scale.py: points within FLIP_BAND of a ReLU tie in the oracle's trace, and points
whose libgfpp and oracle ambient coordinates fall into different cells of some level of the ambient grid (observed, not guessed:
the forward returns the ambient coordinates), where the grid's input gradient jumps.  Each bar is about three times the value
measured on an H100 (in its comment), and each gradient bar at least ten times below the float64 bar it shadows in
tests/test_gpu_field_train_tc.py (0.15, and 0.4 upstream of the ambient grid); each test prints what it measured.
"""
import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF
from helpers import cell_flips, relu_ties
from oracle import field_train as ft
from oracle import field_train_tc as ftc
from oracle import ops

pytestmark = pytest.mark.gpu

FLIP_BAND = 1e-4         # tests/test_gpu_train_scale.py's ReLU-tie band, relative to the layer's largest pre-activation
EXCLUDED_MAX = 0.3       # at most this fraction of the points excluded (measured 24.4 % to 25.0 %, nearly all ReLU ties)
FWD_ABS = 4e-5           # colour / ambient against the rounding oracle, absolute (measured 3.8e-6 to 1.34e-5, the largest at M >= 65 537)
FWD_SIGMA_REL = 5e-4    # sigma, relative to the largest sigma (measured 3.6e-5 to 1.74e-4)
GRAD_L2 = 5e-3           # relative L2 against the rounding oracle: sigma and colour nets, ambient table, code (measured 3.7e-7 to 1.81e-3)
GRAD_L2_UPSTREAM = 1.4e-2  # ... ambient net, position table, cond (measured 1.3e-4 to 4.62e-3); and the faint-only table entries (1.4e-3, 6.4e-3)
UPSTREAM = ("ambient_net.net.0.weight", "ambient_net.net.1.weight", "ambient_net.net.2.weight", "position_embedder.embeddings", "cond")
DET_TAB_REL = 1.5e-5     # table gradients at 262 144 points, run to run: fp32 scatter in free order, more contributions per entry
                         # than tests/test_gpu_field_train_tc.py's 3 001 points (measured 3.2e-6 to 5.2e-6; 1.5e-6 at 3 001)
LOUD, FAINT = 2.0 ** 12, 2.0 ** -40
STEP_OUT_REL = 1e-4      # the steady-state step: rendered outputs against the oracle's, relative to the largest |value| (measured 2.2e-6 to 3.0e-5)

SHAPES = [(3, 4), (2, 0)]   # (ambient_coord_dim, individual_embedding_dim)
FIELD_MS = [3001, 16896, 16897, 65537, 262144]


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _bar(k):
    return GRAD_L2_UPSTREAM if k in UPSTREAM else GRAD_L2


@pytest.fixture(scope="module", params=SHAPES, ids=lambda v: f"amb{v[0]}_ind{v[1]}")
def field_case(request):
    """tests/test_gpu_field_train_tc.py's setup at 262 144 points: points in aabb_train, random upstream gradients, zero at the points
    excluded above."""
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
    model.train_precision = "fp16"
    model = model.cuda()
    g = torch.Generator().manual_seed(7)
    M = FIELD_MS[-1]
    lo, hi = model.aabb_train[:3].cpu(), model.aabb_train[3:].cpu()
    xyzs = lo + (hi - lo) * torch.rand(M, 3, generator=g)
    dirs = F.normalize(torch.randn(M, 3, generator=g), dim=-1)
    cond_feat = model.cal_cond_feat(scn.cond_window(sc.cond, 1, sc.hparams["smo_win_size"]).cuda()).detach().reshape(1, -1).cpu()
    code = state["individual_embeddings"][2].clone() if ind_dim else None
    gs, gc, ga = torch.randn(M, generator=g), torch.randn(M, 3, generator=g), torch.randn(M, amb_dim, generator=g)
    trace = {}
    with torch.no_grad():
        _, _, amb_orc = ftc.field_forward(ft.field_params(state), hp, xyzs, dirs, cond_feat, code, trace=trace)
        _, _, amb_gpu = model.forward(xyzs.cuda(), dirs.cuda(), cond_feat.cuda(), code.cuda() if code is not None else None)
    tie, flip = relu_ties(trace, FLIP_BAND), cell_flips(amb_gpu.cpu(), amb_orc, hp)
    out = tie | flip
    gs[out], gc[out], ga[out] = 0, 0, 0
    frac = float(out.float().mean())
    print(f"[amb {amb_dim}, ind {ind_dim}] {int(tie.sum())} of {M} points at a ReLU tie, {int((flip & ~tie).sum())} more in another ambient "
          f"cell than the oracle's: {100 * frac:.1f} % excluded (bound {100 * EXCLUDED_MAX:.0f} %)")
    assert frac <= EXCLUDED_MAX, frac
    return dict(hp=hp, state=state, model=model, xyzs=xyzs, dirs=dirs, cond=cond_feat, code=code, gs=gs, gc=gc, ga=ga)


def _gpu_field(s, M, up=None):
    m = s["model"]
    m.zero_grad(set_to_none=True)
    gs, gc, ga = up if up is not None else (s["gs"][:M], s["gc"][:M], s["ga"][:M])
    cond = s["cond"].cuda().requires_grad_(True)
    code = s["code"].cuda().requires_grad_(True) if s["code"] is not None else None
    sig, col, amb = m.forward(s["xyzs"][:M].cuda(), s["dirs"][:M].cuda(), cond, code)
    ((sig * gs.cuda()).sum() + (col * gc.cuda()).sum() + (amb * ga.cuda()).sum()).backward()
    grads = {k: p.grad.detach().cpu().clone() for k, p in m.named_parameters() if k in ft.TRAINABLE}
    grads["cond"] = cond.grad.cpu()
    if code is not None:
        grads["code"] = code.grad.cpu()
    torch.cuda.synchronize()
    return (sig.detach().cpu(), col.detach().cpu(), amb.detach().cpu()), grads


def _oracle_field(s, M, up=None):
    """The rounding oracle (fp32, per-tile scale) on the first M points."""
    gs, gc, ga = up if up is not None else (s["gs"][:M], s["gc"][:M], s["ga"][:M])
    p = ft.field_params(s["state"])
    cond = s["cond"].clone().requires_grad_(True)
    code = s["code"].clone().requires_grad_(True) if s["code"] is not None else None
    sig, col, amb = ftc.field_forward(p, s["hp"], s["xyzs"][:M], s["dirs"][:M], cond, code)
    ((sig * gs).sum() + (col * gc).sum() + (amb * ga).sum()).backward()
    grads = {k: p[k].grad for k in ft.TRAINABLE}
    grads["cond"] = cond.grad
    if code is not None:
        grads["code"] = code.grad
    return (sig.detach(), col.detach(), amb.detach()), grads


def _forward_errors(out, ref):
    (sig, col, amb), (rs, rc, ra) = out, ref
    return _rel(sig, rs), (col - rc).abs().max().item(), (amb - ra).abs().max().item()


def _check_grads(tag, g, r):
    bad = []
    for k in r:
        e = _l2(g[k], r[k])
        print(f"{tag} grad {k}: rel L2 to the rounding oracle {e:.2e} (bound {_bar(k):.1e})")
        if not e <= _bar(k):
            bad.append((k, e))
    return bad


@pytest.mark.parametrize("M", FIELD_MS)
def test_field_against_rounding_oracle_across_tiles(field_case, M):
    s = field_case
    out, g = _gpu_field(s, M)
    ref, r = _oracle_field(s, M)
    e = _forward_errors(out, ref)
    print(f"[M {M}] forward: sigma rel {e[0]:.2e} (bound {FWD_SIGMA_REL:.1e}), colour abs {e[1]:.2e}, ambient abs {e[2]:.2e} "
          f"(bound {FWD_ABS:.0e})")
    bad = _check_grads(f"[M {M}]", g, r)
    assert e[0] <= FWD_SIGMA_REL and e[1] <= FWD_ABS and e[2] <= FWD_ABS, e
    assert not bad, bad


def test_faint_tiles_keep_their_bits(field_case):
    """Two tiles per CTA (M = 2 x 132 x 128); the upstream gradients of even tiles times 2^12, of odd tiles times 2^-40.  A kernel
    that chose the power of two per CTA or per call would round every faint tile's dY to zero.  Every gradient against the per-tile
    oracle, and the position-table entries that only faint-tile points reach on their own."""
    s = field_case
    M = 2 * 132 * 128
    odd = (torch.arange(M) // 128) % 2 == 1
    quiet = (torch.arange(M) % 128) < 64             # the first half of each loud tile at 1: the scale is the whole block's

    def up(loud, faint):
        f = torch.where(odd, torch.tensor(faint), torch.where(quiet, torch.tensor(min(loud, 1.0)), torch.tensor(loud)))
        return s["gs"][:M] * f, s["gc"][:M] * f.unsqueeze(1), s["ga"][:M] * f.unsqueeze(1)

    _, g = _gpu_field(s, M, up(LOUD, FAINT))
    _, r = _oracle_field(s, M, up(LOUD, FAINT))
    key = "position_embedder.embeddings"
    _, r_loud = _oracle_field(s, M, up(LOUD, 0.0))
    _, r_faint = _oracle_field(s, M, up(0.0, FAINT))
    only = (r_faint[key] != 0).any(1) & (r_loud[key] == 0).all(1)
    assert all(bool(torch.isfinite(v).all()) for v in g.values())
    e_only = _l2(g[key][only], r[key][only])
    nz = int((g[key][only] != 0).any(1).sum())
    print(f"[M {M}, tiles at 2^12 / 2^-40] {int(only.sum())} position-table entries reached only by faint tiles: {nz} non-zero, rel L2 "
          f"{e_only:.2e} (bound {GRAD_L2_UPSTREAM:.1e}); largest faint-only entry {g[key][only].abs().max().item():.2e}")
    bad = _check_grads(f"[M {M}, spread]", g, r)
    assert int(only.sum()) > 1000 and nz == int((r[key][only] != 0).any(1).sum()), (int(only.sum()), nz)
    assert e_only <= GRAD_L2_UPSTREAM, e_only
    assert not bad, bad


def test_field_backward_deterministic_at_scale(field_case):
    s = field_case
    M = FIELD_MS[-1]
    out1, g1 = _gpu_field(s, M)
    out2, g2 = _gpu_field(s, M)
    assert all(torch.equal(a, b) for a, b in zip(out1, out2))
    worst = 0.0
    for k in g1:
        if k.endswith("embeddings"):
            worst = max(worst, _rel(g1[k], g2[k]))
        else:
            assert torch.equal(g1[k], g2[k]), k
    print(f"[M {M}] outputs and the weight / cond / code gradients bit-identical over two runs; tables run-to-run rel {worst:.2e} "
          f"(bound {DET_TAB_REL:.1e})")
    assert worst <= DET_TAB_REL


def test_field_forward_is_pointwise_across_grid_stride(field_case):
    s = field_case
    (a, b, c), _ = _gpu_field(s, 16896)
    (A, B, C), _ = _gpu_field(s, 65537)
    assert torch.equal(a, A[:16896]) and torch.equal(b, B[:16896]) and torch.equal(c, C[:16896])


# ------------------------------------------------------------------------------------------------ the steady-state training step
def _gradient_mask(out, keep):
    """The field's outputs with their values unchanged and no gradient through the samples where keep is False."""
    return tuple(torch.where(keep.to(o.device).view(-1, *([1] * (o.dim() - 1))), o, o.detach()) for o in out)


def test_steady_state_training_step_fp16(monkeypatch):
    """tests/test_gpu_train_scale.py's steady-state step with train_precision = "fp16": mean_count at about 0.7 x the first step's
    sample count, a buffer of mean_count rounded up to 128 rows, rays past it composite to 0 / the background, every other ray and
    every gradient as in the oracle's render_train with the per-tile rounding oracle as its field.  The GPU field and the oracle see
    the same M-row buffer, so their 128-point tiles hold the same samples.  Samples at a ReLU tie in the oracle's trace, or in another
    ambient cell than the oracle's, pass no gradient to the field in either implementation."""
    ops.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    sc = scn.Scene(H=256, W=256, T=4, torso=False, density_scale=8.0)
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m.conds = sc.cond
    m.train_precision = "fp16"
    m = m.cuda().train()
    fi = sc.frame_inputs(2)
    N = sc.H * sc.W
    args = (fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), None, None)
    with torch.no_grad():
        m.render(*args, index=2, bg_color=fi["bg_color"].cuda(), perturb=False, max_steps=16)
    first = int(m.step_counter[0, 0])
    m.mean_count = int(0.7 * first)
    Mexp = m.mean_count + 128 - m.mean_count % 128
    g = torch.Generator().manual_seed(21)
    coef_rgb, coef_ws, coef_amb = torch.randn(N, 3, generator=g), torch.randn(N, generator=g), torch.randn(N, generator=g)
    with torch.no_grad():
        cond_feat = m.cal_cond_feat(fi["cond"].cuda()).cpu()
    keep = {}
    gpu_forward = m.forward

    def gpu_field(xyzs, dirs, cf, code, **k):
        out = gpu_forward(xyzs, dirs, cf, code, **k)
        tr = {}
        with torch.no_grad():
            _, _, amb = ftc.field_forward(ft.field_params(sc.state), sc.hparams, xyzs.cpu(), dirs.cpu(), cf.detach().cpu(), code.detach().cpu(), trace=tr)
        tie, flip = relu_ties(tr, FLIP_BAND), cell_flips(out[2].detach().cpu(), amb, sc.hparams)
        keep["mask"] = ~(tie | flip)
        keep["counts"] = (int(tie.sum()), int((flip & ~tie).sum()))
        return _gradient_mask(out, keep["mask"])

    monkeypatch.setattr(m, "forward", gpu_field)
    m.zero_grad(set_to_none=True)
    res = m.render(*args, index=2, bg_color=fi["bg_color"].cuda(), perturb=False, max_steps=16)
    ((res["rgb_map"].reshape(-1, 3) * coef_rgb.cuda()).sum() + (res["weights_sum"] * coef_ws.cuda()).sum() + (res["ambient"] * coef_amb.cuda()).sum()).backward()
    torch.cuda.synchronize()

    def oracle_field(p, hp, xyzs, dirs, cf, code):
        return _gradient_mask(ftc.field_forward(p, hp, xyzs, dirs, cf, code), keep["mask"])

    monkeypatch.setattr(ft, "field_forward", oracle_field)
    p = ft.field_params(sc.state)
    emb = sc.state["individual_embeddings"].clone().requires_grad_(True)
    ref = ft.render_train(p, sc.hparams, sc.state, fi["rays_o"], fi["rays_d"], cond_feat, emb[2], fi["bg_color"], sc.density_scale, 16,
                          mean_count=m.mean_count)
    ((ref["rgb_map"].reshape(-1, 3) * coef_rgb).sum() + (ref["weights_sum"] * coef_ws).sum() + (ref["ambient"] * coef_amb).sum()).backward()
    r = {k: p[k].grad for k in ft.TRAINABLE}
    r["code"] = emb.grad[2]
    assert m.step_counter[1].tolist() == [first, N] and res["position"].shape[0] == Mexp
    assert torch.equal(res["position"].detach().cpu(), ref["position"]), "samples differ from the oracle's"
    ro, rd = fi["rays_o"].reshape(-1, 3).contiguous(), fi["rays_d"].reshape(-1, 3).contiguous()
    nears, fars = ops.near_far_from_aabb(ro, rd, sc.state["aabb_train"], sc.hparams["min_near"])
    _, _, _, rays, _ = ops.march_rays_train(ro, rd, 1.0, sc.state["density_bitfield"], 1, sc.hparams["grid_size"], nears, fars, max_steps=16)
    over = (rays[:, 2] > 0) & (rays[:, 1] + rays[:, 2] > Mexp)
    bg = fi["bg_color"].reshape(-1, 3)
    ws, amb, rgb = res["weights_sum"].detach().cpu(), res["ambient"].detach().cpu(), res["rgb_map"].detach().cpu().reshape(-1, 3)
    assert int(over.sum()) > 0
    assert float(ws[over].abs().max()) == 0.0 and float(amb[over].abs().max()) == 0.0 and torch.equal(rgb[over], bg[over].clamp(0, 1))
    e_out = {k: _rel(res[k].detach().cpu().reshape(-1), ref[k].detach().reshape(-1)) for k in ("rgb_map", "weights_sum", "ambient", "depth_map")}
    excl = sum(keep["counts"]) / Mexp
    print(f"[steady step, fp16] first step {first} samples; mean_count {m.mean_count} -> M {Mexp}; {int(over.sum())} of {N} rays overflow; "
          f"{keep['counts'][0]} samples at a ReLU tie, {keep['counts'][1]} more in another ambient cell ({100 * excl:.1f} %); "
          "outputs rel " + ", ".join(f"{k} {v:.2e}" for k, v in e_out.items()) + f" (bound {STEP_OUT_REL:.0e})")
    params = dict(m.named_parameters())
    got = {k: params[k].grad.cpu() for k in ft.TRAINABLE}
    got["code"] = params["individual_embeddings"].grad[2].cpu()
    bad = _check_grads("[steady step, fp16]", got, r)
    assert excl <= EXCLUDED_MAX and max(e_out.values()) <= STEP_OUT_REL, (excl, e_out)
    assert not bad, bad
