"""RADNeRF.frozen_head (gfpp.h section K) pinned exactly, in every precision mode, without a rounding-dependent bar.

Two facts make exact checks possible.  With bound 1 and grid 128 the step is dt_max = 2*sqrt(3)/128 for every max_steps <= 128
(dt_min = min(dt_max, 2*sqrt(3)/max_steps)), so a ray's samples, its jittered start included, do not depend on max_steps; and a
sample's field value depends on its own MMA row only.  So frozen_head(T_thresh=0, max_steps=m) returns the exact fp32 prefix
accumulators (W_m, I_m) of each ray in any mode, and:

- prefix walk: (W_m, I_m) is bit-identical across calls, and frozen once the ray has left the volume (its march_rays_train count);
- termination: frozen_head(T_thresh, max_steps) equals (W_k*, I_k*) bit for bit, k* the first m with 1 - W_m < T_thresh (the
  training rule stops after the sample that takes T below T_thresh), W_max_steps if there is none;
- parity: at T_thresh = 0 frozen_head and the inference renderer (render_frames, same mode, same jitter) differ only by how they
  accumulate T (product against 1 - weights_sum), a few 1e-7.

Beside these: the fp32 mode against the composed fp32 block at the torso step's own settings (dt_gamma 1/256, max_steps 1024, a
two-cascade model), ray counts from 1 to 262 144 with workspace reuse, and in-place edits of every packed parameter."""
import math

import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso
from oracle import torso_train as tt

pytestmark = pytest.mark.gpu

DS = tt.GOLDEN_DS
SEED = 7
# (mlp_precision, GFPP_HEAD_V1): "fp16-v1" is the first-generation fp16 head kernel (k_head_tc<false, false, true>)
MODES = {"fp32": ("fp32", False), "fp16": ("fp16", False), "fp16-v1": ("fp16", True), "robust": ("robust", False),
         "bf16x3": ("bf16x3", False), "bf16": ("bf16", False)}
THRESHOLDS = (1e-4, 1e-2, 0.3)
TERM_DS = 128.0               # at density_scale 8 no ray of these scenes gets below T = 1e-4 within 128 samples
# frozen_head against render_frames at T_thresh = 0 (max-abs over rays with < 128 samples, weights_sum and image): at most
# 3.6e-7 in every mode on an H100 80GB HBM3 at 700 W; the bar is about twice that
PARITY_BAR = 8e-7
FP32_BAR = 1e-5
EXCLUDED_SHARE = 0.01         # rays within m * 2^-20 of T_thresh, where 1 - W_m and the kernel's product T may disagree
TERMINATED_FLOOR = {"golden": 20, "bench256": 1000}   # terminated, non-excluded rays whose extra sample has weight > 0


def _torso_model(state, hp=None):
    m = RADNeRFTorso(hp or may_hparams())
    m.load_state_dict(state, strict=True)
    m.density_scale, m.mlp_precision = DS, "fp32"
    return m.cuda().train()


def _head_model(state, row):
    """A head-only RADNeRF from the same state with code row `row` in row 0, the row the inference renderer folds."""
    m = RADNeRF(may_hparams())
    own = m.state_dict()
    st = {k: v for k, v in state.items() if k in own}
    st["individual_embeddings"] = st["individual_embeddings"].clone()
    st["individual_embeddings"][0] = state["individual_embeddings"][row]
    m.load_state_dict(st, strict=True)
    m.density_scale, m.mlp_precision = DS, "fp32"
    return m.cuda().eval()


class _S:
    pass


@pytest.fixture(scope="module")
def scenes():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    out = {}
    for name, sc in (("golden", tt.golden_scene()), ("bench256", scn.Scene(H=256, W=256, T=4, torso=True, density_scale=DS))):
        s = _S()
        s.sc = sc
        s.m = _torso_model(sc.state)
        s.heads = {row: _head_model(sc.state, row) for row in (0, 2)}
        fi = sc.frame_inputs(tt.GOLDEN_FRAME)
        s.fi = fi
        s.ro, s.rd = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
        with torch.no_grad():
            s.feat = s.m.cal_cond_feat(fi["cond"].cuda())
        assert torch.equal(s.m.aabb_train, s.m.aabb_infer)   # the renderer comparison needs one box for both marchers
        out[name] = s
    return out


@pytest.fixture(params=list(MODES))
def mode(request, monkeypatch):
    prec, v1 = MODES[request.param]
    if v1:
        monkeypatch.setenv("GFPP_HEAD_V1", "1")
    else:
        monkeypatch.delenv("GFPP_HEAD_V1", raising=False)
    return prec


def _fh(m, s, row, prec, perturb, max_steps, T_thresh, dt_gamma=0.0, seed=SEED):
    m.mlp_precision = prec
    try:
        torch.manual_seed(seed)
        return m.frozen_head(s.ro, s.rd, s.feat, m.individual_embeddings[row], perturb=perturb, dt_gamma=dt_gamma, max_steps=max_steps,
                             T_thresh=T_thresh)
    finally:
        m.mlp_precision = "fp32"


def _counts(m, s, perturb, max_steps, dt_gamma=0.0, seed=SEED):
    """Samples per ray of march_rays_train (the third column of its rays table), with the jitter frozen_head draws for `seed`."""
    torch.manual_seed(seed)
    with torch.no_grad():
        nears, fars = train_ops.near_far_from_aabb(s.ro, s.rd, m.aabb_train, m.min_near)
        counter = torch.zeros(2, dtype=torch.int32, device="cuda")
        _, _, _, rays = train_ops.march_rays_train(s.ro, s.rd, m.bound, m.density_bitfield, m.cascade, m.grid_size, nears, fars, counter, 0,
                                                   perturb, 128, True, dt_gamma, max_steps)
    return rays[:, 2].long()


# ------------------------------------------------------------------------------------------------ 1. prefix walk
@pytest.mark.parametrize("scene", ["golden", "bench256"])
@pytest.mark.parametrize("perturb", [False, True])
@pytest.mark.parametrize("row", [0, 2])
def test_prefix_walk_is_deterministic_and_freezes_where_the_ray_leaves(scenes, scene, mode, perturb, row):
    """frozen_head(T_thresh=0, max_steps=m) for m = 1..16 (1..128 on the golden scene): bit-identical on a repeated call; bit-equal
    to the max_steps = M result for every ray with at most m march_rays_train samples; and changed from m - 1 for almost every ray
    that has an m-th sample while it is still transparent (the kernel does shade that sample)."""
    s = scenes[scene]
    m = s.m
    M = 128 if scene == "golden" else 16
    cnt = _counts(m, s, perturb, M)
    ws_M, img_M = _fh(m, s, row, mode, perturb, M, 0.0)
    prev = None
    grew = need = 0
    for k in range(1, M + 1):
        ws, img = _fh(m, s, row, mode, perturb, k, 0.0)
        ws2, img2 = _fh(m, s, row, mode, perturb, k, 0.0)
        assert torch.equal(ws, ws2) and torch.equal(img, img2), f"max_steps={k}: repeated call differs"
        done = cnt <= k
        assert torch.equal(ws[done], ws_M[done]) and torch.equal(img[done], img_M[done]), \
            f"max_steps={k}: a ray with <= {k} samples moved between max_steps {k} and {M}"
        if prev is not None:
            live = (cnt >= k) & (1 - prev[0] > 1e-2)
            changed = (ws != prev[0]) | (img != prev[1]).any(1)
            grew += int((live & changed).sum())
            need += int(live.sum())
        prev = (ws, img)
    print(f"\n[{scene} {mode} perturb={perturb} row={row}] {int((cnt > 0).sum())} rays hit; {grew}/{need} transparent (ray, m) pairs "
          "grew with their m-th sample")
    assert need > 0 and grew >= 0.99 * need


# ------------------------------------------------------------------------------------------------ 2. exact termination
@pytest.mark.parametrize("scene", ["golden", "bench256"])
def test_termination_is_exactly_the_prefix_at_k_star(scenes, scene, mode):
    """frozen_head(T_thresh, max_steps) == (W_k*, I_k*) bit for bit for T_thresh in {1e-4, 1e-2, 0.3} and max_steps in {16, 128},
    with k* the first m where 1 - W_m < T_thresh (W_max_steps if none), over the rays that never come within m * 2^-20 of
    T_thresh.  Walks m upward once (perturb=True, code row 2, density_scale TERM_DS), keeping one running state per threshold, and
    requires a floor of terminated rays whose next sample would have changed the result."""
    s = scenes[scene]
    m = s.m
    m.density_scale = TERM_DS
    try:
        _termination(s, m, scene, mode)
    finally:
        m.density_scale = DS


def _termination(s, m, scene, mode):
    row, N = 2, s.ro.shape[0]
    dev = s.ro.device
    st = {thr: {"k": torch.zeros(N, dtype=torch.long, device=dev), "ws": torch.zeros(N, device=dev), "img": torch.zeros(N, 3, device=dev),
                "excl": torch.zeros(N, dtype=torch.bool, device=dev), "extra": torch.zeros(N, dtype=torch.bool, device=dev)} for thr in THRESHOLDS}
    snap = {}
    for k in range(1, 129):
        ws, img = _fh(m, s, row, mode, True, k, 0.0)
        one_minus = 1 - ws
        for thr, r in st.items():
            after = (r["k"] > 0) & (r["k"] == k - 1)
            r["extra"] |= after & (ws > r["ws"])            # the sample after k* has weight > 0: a late drop would change the result
            alive = r["k"] == 0
            r["excl"] |= alive & ((one_minus - thr).abs() <= k * 2.0 ** -20)
            new = alive & (one_minus < thr)
            r["k"][new] = k
            r["ws"][new] = ws[new]
            r["img"][new] = img[new]
        if k in (16, 128):
            snap[k] = ({thr: {n: t.clone() for n, t in r.items()} for thr, r in st.items()}, ws, img)
    problems = []
    for M, (states, ws_M, img_M) in snap.items():
        for thr, r in states.items():
            term = r["k"] > 0
            exp_ws = torch.where(term, r["ws"], ws_M)
            exp_img = torch.where(term[:, None], r["img"], img_M)
            got_ws, got_img = _fh(m, s, row, mode, True, M, thr)
            keep = ~r["excl"]
            n_excl = int(r["excl"].sum())
            n_term = int((term & keep & (r["k"] < M) & r["extra"]).sum())
            n_bad = int((keep & ((got_ws != exp_ws) | (got_img != exp_img).any(1))).sum())
            print(f"\n[{scene} {mode} T_thresh={thr} max_steps={M}] {int(term.sum())} rays terminate, {n_term} of them checked with a "
                  f"non-zero next sample; {n_excl} excluded ({n_excl / N:.2%}); {n_bad} differ")
            if n_bad or n_excl > EXCLUDED_SHARE * N or n_term < TERMINATED_FLOOR[scene]:
                problems.append((thr, M, n_bad, n_excl, n_term))
    assert not problems, problems


# ------------------------------------------------------------------------------------------------ 3. parity with the inference renderer
@pytest.mark.parametrize("scene", ["golden", "bench256"])
@pytest.mark.parametrize("perturb", [False, True])
@pytest.mark.parametrize("dt_gamma", [0.0, 1 / 256])
@pytest.mark.parametrize("row", [0, 2])
def test_same_precision_parity_with_the_inference_renderer(scenes, scene, mode, perturb, dt_gamma, row):
    """frozen_head(T_thresh=0, max_steps=128) against render_frames(T_thresh=0, max_steps=128, bg_color=0) with the same jitter, in
    the same mode, on the rays with fewer than 128 samples (the others go on into the renderer's second pass).  Code row 2 goes
    through a head model with row 2 copied into row 0."""
    s = scenes[scene]
    m, h = s.m, s.heads[row]
    N = s.ro.shape[0]
    ws_f, img_f = _fh(m, s, row, mode, perturb, 128, 0.0, dt_gamma)
    torch.manual_seed(SEED)
    noise = torch.rand(N, device="cuda") if perturb else None
    h.mlp_precision = mode
    try:
        r = h.render_frames(s.feat.reshape(1, -1), rays_o=s.ro.reshape(1, N, 3), rays_d=s.rd.reshape(1, N, 3), bg_color=0.0, dt_gamma=dt_gamma,
                            max_steps=128, T_thresh=0.0, noise=noise)
    finally:
        h.mlp_precision = "fp32"
    sel = _counts(m, s, perturb, 128, dt_gamma) < 128
    ws_r, img_r = r["weights_sum"].reshape(N), r["rgb_map"].reshape(N, 3)
    e_ws = (ws_f - ws_r)[sel].abs().max().item()
    e_img = (img_f - img_r)[sel].abs().max().item()
    hit = int((ws_r[sel] > 0).sum())
    print(f"\n[{scene} {mode} perturb={perturb} dt_gamma={dt_gamma} row={row}] {int(sel.sum())} rays compared, {hit} hit; "
          f"weights_sum {e_ws:.2e}, image {e_img:.2e}")
    assert hit > 0.05 * N
    assert e_ws <= PARITY_BAR and e_img <= PARITY_BAR


# ------------------------------------------------------------------------------------------------ 4. fp32 at the torso step's settings
def _bound2():
    """A two-cascade (bound 2) torso model: the golden scene's weights, its own bound-2 position grid and aabb, and occupancy in
    both cascades (cascade 1 spans [-2, 2]^3 at half the resolution)."""
    hp = may_hparams(bound=2)
    m = RADNeRFTorso(hp)
    own = m.state_dict()
    src = tt.golden_scene().state
    st = {k: v for k, v in src.items() if k in own and own[k].shape == v.shape and not k.startswith("position_embedder")}
    lay = m.position_embedder.layout
    st["position_embedder.embeddings"] = torch.rand(lay.n_entries, lay.level_dim, generator=torch.Generator().manual_seed(3)) - 0.5
    st["position_embedder.offsets"] = own["position_embedder.offsets"]
    aabb = torch.tensor([-2.0, -1.0, -2.0, 2.0, 1.0, 2.0])
    st["aabb_train"], st["aabb_infer"] = aabb, aabb.clone()
    G = hp["grid_size"]
    grid = torch.cat([scn.ellipsoid_density_grid(G), scn.ellipsoid_density_grid(G, radii=(0.7, 0.45, 0.7))])
    st["density_grid"], st["density_bitfield"] = grid, scn.pack_bitfield(grid)
    for k in own:
        st.setdefault(k, own[k])
    return _torso_model(st, hp)


def _composed(m, ro, rd, feat, code, dt_gamma, max_steps, T_thresh, seed):
    """The no-grad head block of the torso training step on the fp32 training ops."""
    torch.manual_seed(seed)
    with torch.no_grad():
        nears, fars = train_ops.near_far_from_aabb(ro, rd, m.aabb_train, m.min_near)
        counter = torch.zeros(2, dtype=torch.int32, device=ro.device)
        xyzs, dirs, deltas, rays = train_ops.march_rays_train(ro, rd, m.bound, m.density_bitfield, m.cascade, m.grid_size, nears, fars,
                                                              counter, 0, True, 128, True, dt_gamma, max_steps)
        sig, rgb, amb = m(xyzs, dirs, feat, code)
        ws, _, _, img = train_ops.composite_rays_train(m.density_scale * sig, rgb, amb.abs().sum(-1), deltas, rays, T_thresh)
    return ws, img, int(counter[0])


@pytest.mark.parametrize("scene", ["golden", "bench256", "bound2"])
@pytest.mark.parametrize("max_steps", [16, 1024])
def test_fp32_against_composed_at_torso_step_settings(scenes, scene, max_steps):
    """perturb=True, dt_gamma = 1/256, T_thresh = 1e-4, code row 2.  At max_steps 1024 dt_min < t * dt_gamma, so both the step and
    the jitter's step_len(t0) depend on dt_gamma; the bound-2 model marches two cascades."""
    if scene == "bound2":
        m = _bound2()
        sc = scn.Scene(H=128, W=128, T=4, torso=True, density_scale=DS)
        fi = sc.frame_inputs(tt.GOLDEN_FRAME)
        ro, rd = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
        with torch.no_grad():
            feat = m.cal_cond_feat(fi["cond"].cuda())
    else:
        s = scenes[scene]
        m, ro, rd, feat = s.m, s.ro, s.rd, s.feat
    code = m.individual_embeddings[2]
    ws_c, img_c, pts = _composed(m, ro, rd, feat, code, 1 / 256, max_steps, 1e-4, 11)
    torch.manual_seed(11)
    ws_f, img_f = m.frozen_head(ro, rd, feat, code, perturb=True, dt_gamma=1 / 256, max_steps=max_steps, T_thresh=1e-4)
    e_ws, e_img = (ws_f - ws_c).abs().max().item(), (img_f - img_c).abs().max().item()
    hit = int((ws_c > 0).sum())
    print(f"\n[{scene} max_steps={max_steps}] {pts} samples, {hit} rays hit; weights_sum {e_ws:.2e}, image {e_img:.2e}")
    assert hit > 0
    assert e_ws <= FP32_BAR and e_img <= FP32_BAR


# ------------------------------------------------------------------------------------------------ 5. ray counts and workspace reuse
def test_ray_counts_and_workspace_reuse(scenes, mode):
    """One model, consecutive calls that change N (1 .. 262 144) and max_steps, so _frozen_ws is reused and the zeroed histogram and
    counters move with max_steps: each result equals the matching rows of a fresh model's 65 536-ray call."""
    s = scenes["bench256"]
    N = s.ro.shape[0]
    hit = torch.nonzero(_counts(s.m, s, False, 16) > 0).reshape(-1)
    dev = s.ro.device
    picks = {1: hit[len(hit) // 2].reshape(1), 31: torch.arange(31, device=dev) * 2113 % N, 4097: torch.arange(4097, device=dev) * 16 % N,
             N: torch.arange(N, device=dev), 4 * N: torch.arange(4 * N, device=dev) % N}
    calls = [(N, 128), (31, 16), (4 * N, 1024), (1, 4), (4097, 128), (N, 16), (1, 1024), (4 * N, 16)]
    fresh = _torso_model(s.sc.state)
    base = {}
    for ms in sorted({c[1] for c in calls}):
        base[ms] = _fh(fresh, s, 2, mode, False, ms, 1e-4)
    one = _torso_model(s.sc.state)
    one.mlp_precision = mode
    code = one.individual_embeddings[2]
    for n, ms in calls:
        idx = picks[n]
        ws, img = one.frozen_head(s.ro[idx], s.rd[idx], s.feat, code, max_steps=ms, T_thresh=1e-4)
        assert torch.equal(ws, base[ms][0][idx]) and torch.equal(img, base[ms][1][idx]), (n, ms)
    assert int((base[16][0] > 0).sum()) > 0.05 * N


# ------------------------------------------------------------------------------------------------ 6. in-place edits of packed parameters
HEAD_PARAMS = (["individual_embeddings", "position_embedder.embeddings", "ambient_embedder.embeddings"] +
               [f"ambient_net.net.{i}.weight" for i in range(3)] + [f"sigma_net.net.{i}.weight" for i in range(3)] +
               [f"color_net.net.{i}.weight" for i in range(2)])
TORSO_PARAMS = (["torso_embedder.embeddings", "torso_individual_codes"] + [f"torso_deform_net.net.{i}.weight" for i in range(3)] +
                [f"torso_canonicial_net.net.{i}.weight" for i in range(3)])


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("name", HEAD_PARAMS + TORSO_PARAMS)
def test_in_place_edit_of_a_packed_parameter_repacks(scenes, precision, name):
    """After render() and frozen_head() have packed the model, one parameter is edited in place (no invalidate()): the next
    frozen_head() and render() equal those of a model freshly built from the edited state."""
    s = scenes["golden"]
    fi = s.fi
    kw = dict(rays_o=fi["rays_o"].cuda(), rays_d=fi["rays_d"].cuda(), cond=fi["cond"].cuda(), bg_coords=fi["bg_coords"].cuda(),
              poses=fi["poses"].cuda(), bg_color=fi["bg_color"].cuda())

    def run(model):
        model.mlp_precision = precision
        model.train()
        torch.manual_seed(SEED)
        f = model.frozen_head(s.ro, s.rd, s.feat, model.individual_embeddings[2], perturb=True, max_steps=64)
        model.eval()
        r = model.render(**kw)
        model.train()
        return f, r

    m = _torso_model(s.sc.state)
    f0, r0 = run(m)
    p = dict(m.named_parameters())[name]
    with torch.no_grad():
        p.mul_(1.25)
    f1, r1 = run(m)
    fresh = _torso_model({k: v.detach().clone() for k, v in m.state_dict().items()})
    f2, r2 = run(fresh)
    assert torch.equal(f1[0], f2[0]) and torch.equal(f1[1], f2[1]), "frozen_head used a stale pack"
    for k in ("rgb_map", "weights_sum", "torso_alpha_map"):
        assert torch.equal(r1[k], r2[k]), f"render() used a stale pack ({k})"
    assert not torch.equal(r0["rgb_map"], r1["rgb_map"]), "the edit must change the rendered frame"
    if name in HEAD_PARAMS:
        assert not torch.equal(f0[1], f1[1]), "the edit must change the frozen head's image"
