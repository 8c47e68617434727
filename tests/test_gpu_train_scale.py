"""The training path at training-step scale (a step of the May configs marches 65 536 rays into a few hundred thousand samples),
where code paths switch on that no smaller test reaches:

  * the head field (gfpp.h section G, RADNeRF.forward) with several 64-point tiles per backward CTA and a grid-stride forward:
    M = 8 448 (132 CTAs x 64, one tile each), 8 449 (one CTA owns two), 65 537 and 262 144, against oracle/field_train.py;
  * march_rays_train with several 4 096-ray scan tiles, overflow, a non-zero counter at entry, and the scan's limit of 2^24 rays;
  * march_rays_train_backward and composite_rays_train past the grid-stride cap (16 waves of 132 SMs x 8 warps = 16 896 rays), with
    long rays, a T_thresh cut at either end of a 32-sample trip, and rows that overflow M;
  * the grid encoder's training ops at B = 2^20 + 3 (B * L past the grid-stride cap);
  * the steady-state training step: render() after update_extra_state has set mean_count, where M is below the sample count.

References: the C checker (oracle/native_ops.c through oracle/ops.py) and float64 torch.  Bounds are about twice the values measured
on an H100 (DESIGN.md section 3); each test prints what it measured next to its bound.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import _capi, backend_shims
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.config import GridLayout, may_hparams
from genefaceplusplus_b200.renderer import RADNeRF
from helpers import ties
from oracle import field_train as ft
from oracle import ops

pytestmark = pytest.mark.gpu

# the head field: the rule of tests/test_gpu_field_train.py
FWD_REL = 1e-5           # outputs against the fp32 oracle, relative to the largest |value|
GRAD_REL = 1e-4          # gradients against the fp32 oracle, relative to the largest |entry| ...
REF_ROUNDING_FACTOR = 3.0  # ... or no further from the float64 oracle than this times the fp32 oracle is
FLIP_BAND = 1e-4         # points this close to a ReLU tie (relative to the layer's largest pre-activation) carry no upstream gradient
CELL_BAND = 2e-6         # ... and points whose ambient coordinate (the grid's [0,1] input) is this close to a cell face of any level:
                         # libgfpp's and the oracle's ambient coordinates differ in the last bits (measured 4.3e-7 relative), so such a
                         # point can fall into the neighbouring cell, where dy_dx (a per-cell slope of up to 2 048 x the table's steps)
                         # jumps -- one such point moved the ambient net's first-layer gradient by 1.3e-3 at M = 65 537
STEP_GRAD_CAP = 1e-4     # the steady-state step: no gradient further than this from the fp32 oracle, whatever the rule says (measured 3.4e-5)
# compositing
COMP_RAY_BAR = 2e-5      # per-ray bar against the checker (tests/test_gpu_train_ops.py; measured 5.5e-5 on one ray, the 1 024-sample ray,
                         # whose sequential fp32 sums in the checker are the further from float64: 5.0e-5 against libgfpp's 2.6e-5)
COMP_F64_FLOOR = 2e-5    # per-ray distance to float64: at most max(2 x the checker's, this) (measured: no ray over)
KNIFE_EDGE_RAYS = 2      # rays allowed over either bar: a T_thresh crossing within rounding, or a long sum (measured 1 and 0)
MARCH_BWD_REL = 3e-7     # march_rays_train_backward per ray, relative to the sum of |terms| of that ray (measured 1.1e-7)
# grid encoder
GRID_REL = 4e-7          # dy_dx and the input gradient against the checker, relative to the largest |entry| (measured 1.6e-7)
TABLE_REL = 1.2e-6       # table gradient per entry: |d| <= TABLE_REL * S_e + TABLE_ABS, S_e = sum of |w g| reaching the entry: the
TABLE_ABS = 1e-7         # fp32 summation-error scale of the scatter (measured |d| <= 5.4e-7 (S_e + 5e-3))
ADJOINT_REL = 1e-9       # <y, G> - <T, dT> in float64, relative to sum |y G| (measured 2.5e-10)
TV_REL = 2e-5            # TV gradient against the checker, relative to max(1, largest |entry|) (measured 8.3e-6)

SHAPES = [(3, 4), (2, 0)]   # (ambient_coord_dim, individual_embedding_dim)
FIELD_MS = [8448, 8449, 65537, 262144]


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _rm():
    return backend_shims.make_modules()["_raymarching_face"]


# ------------------------------------------------------------------------------------------------ 1. head field across CTA tiles

@pytest.fixture(scope="module", params=SHAPES, ids=lambda v: f"amb{v[0]}_ind{v[1]}")
def field_case(request):
    """tests/test_gpu_field_train.py's setup at 262 144 points: points in aabb_train, random upstream gradients, none at a ReLU tie."""
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
    M = FIELD_MS[-1]
    lo, hi = model.aabb_train[:3].cpu(), model.aabb_train[3:].cpu()
    xyzs = lo + (hi - lo) * torch.rand(M, 3, generator=g)
    dirs = F.normalize(torch.randn(M, 3, generator=g), dim=-1)
    cond_feat = model.cal_cond_feat(scn.cond_window(sc.cond, 1, sc.hparams["smo_win_size"]).cuda()).detach().reshape(1, -1)
    code = state["individual_embeddings"][2].clone() if ind_dim else None
    gs, gc, ga = torch.randn(M, generator=g), torch.randn(M, 3, generator=g), torch.randn(M, amb_dim, generator=g)
    trace = {}
    _, _, amb = ft.field_forward(ft.field_params(state), hp, xyzs, dirs, cond_feat.cpu(), code, trace=trace)
    tie, face = ties(trace, amb, hp, FLIP_BAND, CELL_BAND)
    gs[tie | face], gc[tie | face], ga[tie | face] = 0, 0, 0
    print(f"[amb {amb_dim}, ind {ind_dim}] {int(tie.sum())} of {M} points at a ReLU tie, {int((face & ~tie).sum())} more at an ambient cell face")
    return dict(hp=hp, state=state, model=model, xyzs=xyzs, dirs=dirs, cond=cond_feat.cpu(), code=code, gs=gs, gc=gc, ga=ga)


def _gpu_field(s, M):
    m = s["model"]
    m.zero_grad(set_to_none=True)
    cond = s["cond"].cuda().requires_grad_(True)
    code = s["code"].cuda().requires_grad_(True) if s["code"] is not None else None
    sig, col, amb = m.forward(s["xyzs"][:M].cuda(), s["dirs"][:M].cuda(), cond, code)
    ((sig * s["gs"][:M].cuda()).sum() + (col * s["gc"][:M].cuda()).sum() + (amb * s["ga"][:M].cuda()).sum()).backward()
    grads = {k: p.grad.detach().cpu().clone() for k, p in m.named_parameters() if k in ft.TRAINABLE}
    grads["cond"] = cond.grad.cpu()
    if code is not None:
        grads["code"] = code.grad.cpu()
    torch.cuda.synchronize()
    return (sig.detach().cpu(), col.detach().cpu(), amb.detach().cpu()), grads


def _oracle_field(s, M, dtype):
    p = ft.field_params(s["state"], dtype)
    cond = s["cond"].clone().to(dtype).requires_grad_(True)
    code = s["code"].clone().to(dtype).requires_grad_(True) if s["code"] is not None else None
    sig, col, amb = ft.field_forward(p, s["hp"], s["xyzs"][:M], s["dirs"][:M].to(dtype), cond, code)
    ((sig * s["gs"][:M].to(dtype)).sum() + (col * s["gc"][:M].to(dtype)).sum() + (amb * s["ga"][:M].to(dtype)).sum()).backward()
    grads = {k: p[k].grad for k in ft.TRAINABLE}
    grads["cond"] = cond.grad
    if code is not None:
        grads["code"] = code.grad
    return (sig.detach(), col.detach(), amb.detach()), grads


def _check_grads(tag, g, r, r64, cap=None):
    for k in r:
        e = _rel(g[k], r[k])
        e_gpu, e_orc = _rel(g[k].double(), r64[k].double()), _rel(r[k].double(), r64[k].double())
        ok = e <= GRAD_REL or e_gpu <= REF_ROUNDING_FACTOR * e_orc
        print(f"{tag} grad {k}: rel {e:.2e} (bound {GRAD_REL:.0e}); to float64: libgfpp {e_gpu:.2e}, fp32 oracle {e_orc:.2e} "
              f"(bound {REF_ROUNDING_FACTOR:g}x)" + ("" if cap is None else f"; cap {cap:.0e}"))
        assert ok and (cap is None or e <= cap), (k, e, e_gpu, e_orc)


@pytest.mark.parametrize("M", FIELD_MS)
def test_field_against_oracle_across_tiles(field_case, M):
    s = field_case
    (sig, col, amb), g = _gpu_field(s, M)
    (rs, rc, ra), r = _oracle_field(s, M, torch.float32)
    _, r64 = _oracle_field(s, M, torch.float64)
    e = [_rel(sig, rs), _rel(col, rc), _rel(amb, ra)]
    print(f"[M {M}] forward rel err sigma {e[0]:.2e} colour {e[1]:.2e} ambient {e[2]:.2e} (bound {FWD_REL:.0e})")
    assert max(e) <= FWD_REL, e
    _check_grads(f"[M {M}]", g, r, r64)


def test_field_backward_deterministic_at_scale(field_case):
    s = field_case
    M = FIELD_MS[-1]
    out1, g1 = _gpu_field(s, M)
    out2, g2 = _gpu_field(s, M)
    assert all(torch.equal(a, b) for a, b in zip(out1, out2))
    for k in g1:
        if not k.endswith("embeddings"):
            assert torch.equal(g1[k], g2[k]), k
    print(f"[M {M}] outputs and the weight / cond / code gradients bit-identical over two runs")


def test_field_forward_is_pointwise_across_grid_stride(field_case):
    s = field_case
    (a, b, c), _ = _gpu_field(s, 8448)
    (A, B, C), _ = _gpu_field(s, 65537)
    assert torch.equal(a, A[:8448]) and torch.equal(b, B[:8448]) and torch.equal(c, C[:8448])


# ------------------------------------------------------------------------------------------------ 2. march_rays_train at scale
_FRAMES = {}


def _frame_rays(H):
    """rays_o, rays_d, nears, fars (CPU) of frame 1 of an H x H scene, and its bitfield."""
    if H not in _FRAMES:
        sc = scn.Scene(H=H, W=H, T=2, torso=False)
        fi = sc.frame_inputs(1)
        ro, rd = fi["rays_o"].reshape(-1, 3).contiguous(), fi["rays_d"].reshape(-1, 3).contiguous()
        nears, fars = ops.near_far_from_aabb(ro, rd, sc.state["aabb_infer"], 0.05)
        _FRAMES[H] = (ro, rd, nears, fars, sc.state["density_bitfield"])
    return _FRAMES[H]


def _march_inputs(N):
    """N rays: a 256^2 or 512^2 frame, or a crop of the 256^2 frame around its centre for the odd sizes."""
    H = 512 if N > 65536 else 256
    ro, rd, nears, fars, bits = _frame_rays(H)
    a = (H * H - N) // 2
    return ro[a:a + N].contiguous(), rd[a:a + N].contiguous(), nears[a:a + N].contiguous(), fars[a:a + N].contiguous(), bits


def _gpu_march(ro, rd, nears, fars, bits, noises, M, counter0, max_steps, dt_gamma):
    N = ro.shape[0]
    xyzs, dirs, deltas = torch.zeros(M, 3, device="cuda"), torch.zeros(M, 3, device="cuda"), torch.zeros(M, 2, device="cuda")
    rays = torch.full((N, 3), -7, dtype=torch.int32, device="cuda")
    counter = counter0.clone().cuda()
    _rm().march_rays_train(ro.cuda(), rd.cuda(), bits.cuda(), 1.0, dt_gamma, max_steps, N, 1, 128, M, nears.cuda(), fars.cuda(), xyzs, dirs, deltas,
                           rays, counter, noises.cuda())
    torch.cuda.synchronize()
    return xyzs.cpu(), dirs.cpu(), deltas.cpu(), rays.cpu(), counter.cpu()


def _cut_ray(rays):
    """A ray with >= 2 samples in scan tile min(8, last) (or anywhere, failing that): an M of its offset + 1 cuts inside it."""
    N = rays.shape[0]
    tile = min(8, (N - 1) // 4096)
    cand = torch.nonzero(rays[:, 2] >= 2).view(-1)
    inside = cand[(cand >= tile * 4096) & (cand < (tile + 1) * 4096)]
    n = int((inside if inside.numel() else cand)[inside.numel() // 2 if inside.numel() else cand.numel() // 2])
    return n, n // 4096


@pytest.mark.parametrize("noise", [False, True], ids=["noise_off", "noise_on"])
@pytest.mark.parametrize("N", [4095, 4097, 65536, 262144])
def test_march_rays_train_at_scale(N, noise):
    ops.build()
    ro, rd, nears, fars, bits = _march_inputs(N)
    max_steps, dt_gamma = 16, 1 / 256
    noises = torch.rand(N, generator=torch.Generator().manual_seed(N)) if noise else torch.zeros(N)
    M = N * max_steps
    ref = ops.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, noises=noises, dt_gamma=dt_gamma, max_steps=max_steps)
    zero = torch.zeros(2, dtype=torch.int32)
    got = _gpu_march(ro, rd, nears, fars, bits, noises, M, zero, max_steps, dt_gamma)
    names = ("xyzs", "dirs", "deltas", "rays", "counter")
    for nm, a, b in zip(names, got, ref):
        assert torch.equal(a, b), nm
    again = _gpu_march(ro, rd, nears, fars, bits, noises, M, zero, max_steps, dt_gamma)
    assert all(torch.equal(a, b) for a, b in zip(again, got)), "two runs differ"
    # a counter that is not zero at entry (offsets start at K) and an M that cuts inside one ray of scan tile 8
    K, c1 = 12345, 7
    pre = torch.tensor([K, c1], dtype=torch.int32)
    _, _, _, r_k, _ = ops.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, noises=noises, dt_gamma=dt_gamma, max_steps=max_steps,
                                           counter=pre.clone())
    n_cut, tile = _cut_ray(r_k)
    Mc = int(r_k[n_cut, 1]) + 1
    ref_c = ops.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, M=Mc, noises=noises, dt_gamma=dt_gamma, max_steps=max_steps,
                                 counter=pre.clone())
    got_c = _gpu_march(ro, rd, nears, fars, bits, noises, Mc, pre, max_steps, dt_gamma)
    for nm, a, b in zip(names, got_c, ref_c):
        assert torch.equal(a, b), ("counter K, overflow", nm)
    over = int(((r_k[:, 1] + r_k[:, 2] > Mc) & (r_k[:, 2] > 0)).sum())
    print(f"[N {N}, noise {noise}] {int(ref[4][0])} samples, bit-exact with the checker and run to run; counter [{K}, {c1}] at entry with "
          f"M = {Mc} (cut in ray {n_cut}, scan tile {tile}, {over} rays overflow): bit-exact")


def test_march_rays_train_scan_limit():
    """N = 2^24 rays (the 512^2 frame tiled 64 times, max_steps 4, M about 2^20): 4 096 tile sums in the one CTA of k_scan_tops.
    N = 2^24 + 1 is refused before anything is written."""
    ops.build()
    ro, rd, nears, fars, bits = _frame_rays(512)
    reps = (1 << 24) // ro.shape[0]
    N, max_steps, M = 1 << 24, 4, 1 << 20
    K, c1 = 1000, 3
    dev = "cuda"
    ro_d, rd_d = ro.to(dev).repeat(reps, 1), rd.to(dev).repeat(reps, 1)
    nears_d, fars_d = nears.to(dev).repeat(reps), fars.to(dev).repeat(reps)
    noises = torch.zeros(N, device=dev)
    xyzs, dirs, deltas = torch.zeros(M, 3, device=dev), torch.zeros(M, 3, device=dev), torch.zeros(M, 2, device=dev)
    rays = torch.full((N, 3), -7, dtype=torch.int32, device=dev)
    counter = torch.tensor([K, c1], dtype=torch.int32, device=dev)
    _rm().march_rays_train(ro_d, rd_d, bits.to(dev), 1.0, 0.0, max_steps, N, 1, 128, M, nears_d, fars_d, xyzs, dirs, deltas, rays, counter, noises)
    torch.cuda.synchronize()
    rays_c = rays.cpu()
    counts = rays_c[:, 2].long()
    expect = K + torch.cumsum(counts, 0) - counts
    total = int(counts.sum())
    assert torch.equal(rays_c[:, 0], torch.arange(N, dtype=torch.int32))
    assert torch.equal(rays_c[:, 1].long(), expect)
    assert counter.cpu().tolist() == [K + total, c1 + N]
    # a strided subset of rays against the checker run on that subset alone
    sub = torch.arange(0, N, 1021)
    src = sub % ro.shape[0]
    sub_ro, sub_rd, sub_n, sub_f = ro[src].contiguous(), rd[src].contiguous(), nears[src].contiguous(), fars[src].contiguous()
    xr, dr, lr, rr, _ = ops.march_rays_train(sub_ro, sub_rd, 1.0, bits, 1, 128, sub_n, sub_f, max_steps=max_steps)
    assert torch.equal(rr[:, 2], rays_c[sub, 2])
    xg, dg, lg = xyzs.cpu(), dirs.cpu(), deltas.cpu()
    compared = 0
    for j, n in enumerate(sub.tolist()):
        o, k = int(rays_c[n, 1]), int(rays_c[n, 2])
        if k == 0 or o + k > M:
            continue
        q = int(rr[j, 1])
        assert torch.equal(xg[o:o + k], xr[q:q + k]) and torch.equal(dg[o:o + k], dr[q:q + k]) and torch.equal(lg[o:o + k], lr[q:q + k]), n
        compared += 1
    assert compared > 100
    print(f"[N 2^24] {total} samples (M {M}); offsets = {K} + int64 exclusive cumsum, counter {counter.cpu().tolist()}; "
          f"{compared} rays of the strided subset bit-exact with the checker")
    del xyzs, dirs, deltas
    # N = 2^24 + 1: GFPP_ERR_UNSUPPORTED, nothing written
    N1 = N + 1
    ro1, rd1 = torch.cat([ro_d, ro_d[:1]]), torch.cat([rd_d, rd_d[:1]])
    del ro_d, rd_d
    n1, f1, z1 = torch.cat([nears_d, nears_d[:1]]), torch.cat([fars_d, fars_d[:1]]), torch.zeros(N1, device=dev)
    del rays
    rays1 = torch.full((N1, 3), -7, dtype=torch.int32, device=dev)
    small = 4096
    x1, d1, l1 = torch.full((small, 3), 5.0, device=dev), torch.full((small, 3), 5.0, device=dev), torch.full((small, 2), 5.0, device=dev)
    cnt1 = torch.tensor([K, c1], dtype=torch.int32, device=dev)
    L = _capi.lib()
    need = L.gfpp_march_rays_train_scratch_bytes(N1)
    scratch = torch.zeros(need, dtype=torch.uint8, device=dev)
    P = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    rc = L.gfpp_march_rays_train(P(ro1), P(rd1), P(bits.to(dev)), ctypes.c_float(1.0), ctypes.c_float(0.0), max_steps, N1, 1, 128, small, P(n1), P(f1),
                                 P(x1), P(d1), P(l1), P(rays1), P(cnt1), P(z1), P(scratch), need, _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == -4, rc   # GFPP_ERR_UNSUPPORTED
    assert bool((rays1 == -7).all()) and cnt1.cpu().tolist() == [K, c1] and bool((scratch == 0).all())
    assert bool((x1 == 5.0).all()) and bool((d1 == 5.0).all()) and bool((l1 == 5.0).all())
    print(f"[N 2^24 + 1] rc {rc} ({L.gfpp_last_error().decode()}); nothing written")


# ------------------------------------------------------------------------------------------------ 3. march_rays_train_backward
def _samples_of(rays, M):
    """(rows with samples inside M [N] bool, the row of each of their samples, the sample's index), through the rays table."""
    off, ns = rays[:, 1].long(), rays[:, 2].long()
    ok = (ns > 0) & (off + ns <= M)
    n_of = torch.repeat_interleave(torch.arange(rays.shape[0])[ok], ns[ok])
    s_of = torch.repeat_interleave(off[ok], ns[ok]) + torch.arange(int(ns[ok].sum())) - torch.repeat_interleave(torch.cumsum(ns[ok], 0) - ns[ok], ns[ok])
    return ok, n_of, s_of


@pytest.mark.parametrize("N", [65536, 262144])
def test_march_rays_train_backward_at_scale(N):
    ops.build()
    ro, rd, nears, fars, bits = _march_inputs(N)
    max_steps = 16
    noises = torch.rand(N, generator=torch.Generator().manual_seed(5))
    xyzs, _, deltas, rays, counter = _gpu_march(ro, rd, nears, fars, bits, noises, N * max_steps, torch.zeros(2, dtype=torch.int32), max_steps, 1 / 256)
    m = int(counter[0])
    n_cut, _ = _cut_ray(rays)
    Mc = int(rays[n_cut, 1]) + 1                       # rows from ray n_cut on overflow: their gradient rows stay zero
    g = torch.Generator().manual_seed(6)
    gx, gd = torch.randn(Mc, 3, generator=g), torch.randn(Mc, 3, generator=g)
    dl = deltas[:Mc].contiguous()
    go, gdd = torch.zeros(N, 3, device="cuda"), torch.zeros(N, 3, device="cuda")
    _rm().march_rays_train_backward(gx.cuda(), gd.cuda(), rays.cuda(), dl.cuda(), N, Mc, go, gdd)
    torch.cuda.synchronize()
    go, gdd = go.cpu().double(), gdd.cpu().double()
    # float64 per-ray segment sums through the rays table (row n gets ray n's samples, as the reference does)
    live, n_of, s_of = _samples_of(rays, Mc)
    t = dl[s_of, 1].double().unsqueeze(1)
    tx, td = gx[s_of].double(), gx[s_of].double() * t + gd[s_of].double()
    ref_o = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, n_of, tx)
    ref_d = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, n_of, td)
    sc_o = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, n_of, tx.abs())
    sc_d = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, n_of, (gx[s_of].double() * t).abs() + gd[s_of].double().abs())
    e_o = ((go - ref_o).abs() / sc_o.clamp_min(1e-30))[live].max().item()
    e_d = ((gdd - ref_d).abs() / sc_d.clamp_min(1e-30))[live].max().item()
    print(f"[N {N}] {m} samples, M {Mc}: per-ray error to float64 / sum|terms|: rays_o {e_o:.2e}, rays_d {e_d:.2e} (bound {MARCH_BWD_REL:.0e}); "
          f"{int((~live & (rays[:, 2] > 0)).sum())} overflowed rows stay 0")
    assert e_o <= MARCH_BWD_REL and e_d <= MARCH_BWD_REL
    assert float(go[~live].abs().max()) == 0.0 and float(gdd[~live].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ 4. composite_rays_train
def _long_segments(N=100003, seed=3):
    """Lengths U(0,16) plus ~1 % long rays of 100..1 024 samples, three constructed rays -- cut at lane 31 of trip 2 (sample 95), at
    lane 0 of trip 3 (sample 96), never cut (1 024 samples of tiny sigma) -- a permuted rays[:,0], and an M that leaves the last ~5 %
    of rows with offset + num_steps > M (one of them cut inside)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, 16, (N,), generator=g)
    longs = torch.randperm(N, generator=g)[: N // 100]
    lens[longs] = torch.randint(100, 1025, (longs.numel(),), generator=g)
    special = [11, 12, 13]
    lens[special] = torch.tensor([200, 200, 1024])
    offs = torch.cumsum(lens, 0) - lens
    total = int(lens.sum())
    sig = torch.rand(total, generator=g) * 6
    rgb = torch.rand(total, 3, generator=g)
    amb = torch.rand(total, generator=g)
    dt = torch.rand(total, generator=g) * 0.05 + 0.01
    deltas = torch.stack([dt, torch.rand(total, generator=g) * 3 + 2], 1)
    for n, cut in zip(special, [95, 96, None]):
        o, k = int(offs[n]), int(lens[n])
        sig[o:o + k] = 1e-3 if cut is None else 0.01
        if cut is not None:
            sig[o + cut] = 1e3
    first_over = int(N * 0.95)
    while lens[first_over] < 2:
        first_over += 1
    M = int(offs[first_over]) + 1
    perm = torch.randperm(N, generator=g).int()
    rays = torch.stack([perm, offs.int(), lens.int()], 1).contiguous()
    return rays, M, sig[:M].contiguous(), rgb[:M].contiguous(), amb[:M].contiguous(), deltas[:M].contiguous(), special


def _composite_f64(sig, rgb, amb, deltas, rays, M, T_thresh, gws, gas, gim):
    """The rendering formula with its early break in float64, bucketed by ray length; forward per ray index, backward per sample."""
    N = rays.shape[0]
    idx, off, ns = rays[:, 0].long(), rays[:, 1].long(), rays[:, 2].long()
    ws, asum, depth, image = torch.zeros(N, dtype=torch.float64), torch.zeros(N, dtype=torch.float64), torch.zeros(N, dtype=torch.float64), torch.zeros(N, 3, dtype=torch.float64)
    gs, gr, ga = torch.zeros(M, dtype=torch.float64), torch.zeros(M, 3, dtype=torch.float64), torch.zeros(M, dtype=torch.float64)
    ok = (ns > 0) & (off + ns <= M)
    lo = 0
    for hi in (16, 32, 64, 128, 256, 512, 1024):
        rows = torch.nonzero(ok & (ns > lo) & (ns <= hi)).view(-1)
        lo = hi
        if rows.numel() == 0:
            continue
        k = torch.arange(hi)
        have = k.unsqueeze(0) < ns[rows].unsqueeze(1)
        p = (off[rows].unsqueeze(1) + k.unsqueeze(0)).clamp(max=M - 1)
        s_, dt_, tt = sig.double()[p], deltas.double()[p, 0], deltas.double()[p, 1]
        c = rgb.double()[p]
        alpha = torch.where(have, 1 - torch.exp(-s_ * dt_), torch.zeros_like(s_))
        T_after = torch.cumprod(1 - alpha, 1)
        T_before = torch.cat([torch.ones(rows.numel(), 1, dtype=torch.float64), T_after[:, :-1]], 1)
        live = have & (T_before >= T_thresh)           # T never grows: every earlier sample left T >= T_thresh
        w = torch.where(live, alpha * T_before, torch.zeros_like(alpha))
        cum = torch.cumsum(w.unsqueeze(-1) * c, 1)
        r = idx[rows]
        ws[r] = w.sum(1)
        asum[r] = torch.where(live, amb.double()[p], torch.zeros_like(alpha)).sum(1)
        depth[r] = (w * tt).sum(1)
        image[r] = cum[:, -1]
        gi = gim.double()[r].unsqueeze(1)
        g_s = dt_ * ((gi * (T_after.unsqueeze(-1) * c - (image[r].unsqueeze(1) - cum))).sum(-1) + gws.double()[r].unsqueeze(1) * (1 - ws[r].unsqueeze(1)))
        pl = p[live]
        gs[pl] = g_s[live]
        gr[pl] = (gi * w.unsqueeze(-1))[live]
        ga[pl] = gas.double()[r].unsqueeze(1).expand_as(w)[live]
    return (ws, asum, depth, image), (gs, gr, ga)


def _per_ray(err_samples, rays, M):
    """max over each ray's samples -> [N] (rows that overflow M: 0)."""
    _, n_of, s_of = _samples_of(rays, M)
    return torch.zeros(rays.shape[0], dtype=torch.float64).scatter_reduce_(0, n_of, err_samples.double()[s_of], "amax")


def test_composite_rays_train_past_the_grid_cap():
    ops.build()
    T_thresh = 1e-4
    rays, M, sig, rgb, amb, deltas, special = _long_segments()
    N = rays.shape[0]
    g = torch.Generator().manual_seed(9)
    gws, gas, gim = torch.randn(N, generator=g), torch.randn(N, generator=g), torch.randn(N, 3, generator=g)
    rm = _rm()
    dev = "cuda"
    d_sig, d_rgb, d_amb, d_dl, d_rays = sig.to(dev), rgb.to(dev), amb.to(dev), deltas.to(dev), rays.to(dev)

    def fwd():
        out = [torch.full((N,), float("nan"), device=dev) for _ in range(3)] + [torch.full((N, 3), float("nan"), device=dev)]
        rm.composite_rays_train_forward(d_sig, d_rgb, d_amb, d_dl, d_rays, M, N, T_thresh, *out)
        torch.cuda.synchronize()
        return out

    def bwd(out, fill):
        grads = [torch.full((M,), fill, device=dev), torch.full((M, 3), fill, device=dev), torch.full((M,), fill, device=dev)]
        rm.composite_rays_train_backward(gws.to(dev), gas.to(dev), gim.to(dev), d_sig, d_rgb, d_amb, d_dl, d_rays, out[0], out[1], out[3], M, N,
                                         T_thresh, *grads)
        torch.cuda.synchronize()
        return [t.cpu() for t in grads]

    out = fwd()
    g1 = bwd(out, 0.0)
    out_c = [t.cpu() for t in out]
    assert all(torch.equal(a.cpu(), b) for a, b in zip(fwd(), out_c)) and all(torch.equal(a, b) for a, b in zip(bwd(out, 0.0), g1)), "two runs differ"
    # overflowed rows: outputs exactly 0, gradient slots untouched
    idx, off, ns = rays[:, 0].long(), rays[:, 1].long(), rays[:, 2].long()
    over = (ns > 0) & (off + ns > M)
    assert 0.04 * N < int(over.sum()) < 0.06 * N
    assert all(float(t[idx[over]].abs().max()) == 0.0 for t in out_c)
    g7 = bwd(out, 7.0)
    cut_row = int(torch.nonzero(over & (off < M)).view(-1)[0])
    tail = slice(int(off[cut_row]), M)
    assert all(bool((t[tail] == 7.0).all()) for t in g7), "the slots of a row that overflows M were written"
    assert all(bool(((a == b) | ((a == 0) & (b == 7.0))).all()) for a, b in zip(g1, g7))
    # against the checker: the per-ray bar, knife-edge rays counted
    ws, asum, depth, image = ops.composite_rays_train_forward(sig, rgb, amb, deltas, rays, T_thresh)
    gs, gr, ga = ops.composite_rays_train_backward(gws, gas, gim, sig, rgb, amb, deltas, rays, ws, asum, image, T_thresh)

    def fwd_err(o):
        return torch.stack([(o[0] - ws.double()).abs()[idx], (o[1] - asum.double()).abs()[idx] * 0.1, (o[2] - depth.double()).abs()[idx],
                            (o[3] - image.double()).abs().max(-1).values[idx]]).max(0).values

    def bwd_err(a, b):
        return torch.stack([_per_ray((a[0] - b[0]).abs() / max(1.0, b[0].abs().max().item()), rays, M), _per_ray((a[1] - b[1]).abs().max(-1).values, rays, M),
                            _per_ray((a[2] - b[2]).abs(), rays, M)]).max(0).values

    gpu_o = [t.double() for t in out_c]
    e_chk = torch.maximum(fwd_err(gpu_o), bwd_err([t.double() for t in g1], [gs.double(), gr.double(), ga.double()]))
    bad = (e_chk > COMP_RAY_BAR).nonzero().view(-1)
    # against float64
    (w64, a64, d64, i64), (gs64, gr64, ga64) = _composite_f64(sig, rgb, amb, deltas, rays, M, T_thresh, gws, gas, gim)
    f64 = [w64, a64, d64, i64]

    def err64(o, gr_):
        e = torch.stack([(o[0] - f64[0]).abs()[idx], (o[1] - f64[1]).abs()[idx] * 0.1, (o[2] - f64[2]).abs()[idx],
                         (o[3] - f64[3]).abs().max(-1).values[idx]]).max(0).values
        return torch.maximum(e, bwd_err([t.double() for t in gr_], [gs64, gr64, ga64]))

    e_gpu64 = err64(gpu_o, g1)
    e_chk64 = err64([ws.double(), asum.double(), depth.double(), image.double()], [gs, gr, ga])
    bad64 = (e_gpu64 > torch.clamp(2 * e_chk64, min=COMP_F64_FLOOR)).nonzero().view(-1)
    print(f"[composite N {N}, M {M}, {int(ns.sum())} samples, longest {int(ns.max())}] vs checker: max per-ray {e_chk.max().item():.2e}, "
          f"rays over {COMP_RAY_BAR:.0e}: {bad.numel()}; to float64: libgfpp max {e_gpu64.max().item():.2e}, checker max {e_chk64.max().item():.2e}, "
          f"rays over max(2x checker, {COMP_F64_FLOOR:.0e}): {bad64.numel()} (allowed {KNIFE_EDGE_RAYS} each); {int(over.sum())} rows overflow M")
    assert bad.numel() <= KNIFE_EDGE_RAYS and bad64.numel() <= KNIFE_EDGE_RAYS, (bad.tolist(), bad64.tolist())
    # the constructed rays: the cut where it was built, the same in libgfpp, the checker and float64
    for n, cut in zip(special, [95, 96, None]):
        o, k = int(off[n]), int(ns[n])
        last = k - 1 if cut is None else cut
        for grads in (g1, [gs, gr, ga]):
            assert bool((grads[1][o:o + last + 1].abs().sum(-1) > 0).all()) and bool((grads[1][o + last + 1:o + k] == 0).all()), (n, cut)
        assert n not in bad64.tolist()


# ------------------------------------------------------------------------------------------------ 5. grid encoder training ops
GRID_CASES = [(3, 1, 0), (2, 1, 0), (3, 0, 1)]   # (D, gridtype, interp): tiled 3-D at the position layout, tiled 2-D, hash 3-D smoothstep


@pytest.mark.parametrize("D,gridtype,interp", GRID_CASES, ids=["tiled3d_pos", "tiled2d", "hash3d_smooth"])
def test_grid_training_ops_past_the_grid_cap(D, gridtype, interp):
    ops.build()
    if gridtype == 1:
        lay = GridLayout(D, log2_hashmap_size=16, desired_resolution=2048, gridtype="tiled")
    else:
        lay = GridLayout(D, log2_hashmap_size=14, desired_resolution=512, gridtype="hash", interpolation="smoothstep")
    offsets = torch.from_numpy(np.asarray(lay.offsets, dtype=np.int32))
    L = offsets.numel() - 1
    g = torch.Generator().manual_seed(100 + D * 10 + gridtype)
    table = torch.rand(int(offsets[-1]), 2, generator=g) - 0.5
    B = (1 << 20) + 3
    x = torch.rand(B, D, generator=g) * 0.98 + 0.01
    G = torch.randn(B, L * 2, generator=g)
    dydx_ref = ops.grid_encode_dydx(x, table, offsets, lay.per_level_scale, 16, gridtype, False, interp)
    ge_ref, gi_ref = ops.grid_encode_backward(G, x, table, offsets, lay.per_level_scale, 16, gridtype, False, interp, dy_dx=dydx_ref)
    S_e, _ = ops.grid_encode_backward(G.abs(), x, table, offsets, lay.per_level_scale, 16, gridtype, False, interp)
    # libgfpp: forward with dy_dx, backward (table and input gradient) through the wrapper's own buffers
    ge_mod = backend_shims.make_modules()["_gridencoder"]
    S = float(np.log2(lay.per_level_scale))
    xd, td = x.cuda(), table.cuda()
    y = torch.empty(L, B, 2, device="cuda")
    dy = torch.empty(B, L * D * 2, device="cuda")
    ge_mod.grid_encode_forward(xd, td, offsets.cuda(), y, B, D, 2, L, S, 16, dy, gridtype, False, interp)
    grad = G.view(B, L, 2).permute(1, 0, 2).contiguous().cuda()
    ge, gi = torch.zeros_like(td), torch.zeros(B, D, device="cuda")
    ge_mod.grid_encode_backward(grad, xd, td, offsets.cuda(), ge, B, D, 2, L, S, 16, dy, gi, gridtype, False, interp)
    torch.cuda.synchronize()
    dy, gi, ge = dy.cpu().view(B, L, D, 2), gi.cpu(), ge.cpu()
    e_dy, e_gi = _rel(dy, dydx_ref), _rel(gi, gi_ref)
    tab_excess = ((ge - ge_ref).abs() - (TABLE_REL * S_e + TABLE_ABS)).max().item()
    tab_ratio = ((ge - ge_ref).abs() / (S_e + TABLE_ABS / TABLE_REL)).max().item()
    # adjoint identity of the linear map T -> y:  <y, G> = <T, dL/dT>
    yG = y.cpu().permute(1, 0, 2).reshape(B, L * 2).double() * G.double()
    adj = abs(yG.sum().item() - (table.double() * ge.double()).sum().item()) / yG.abs().sum().item()
    # total variation gradient of the cells the same inputs fall into
    xb = x * 2 - 1                                     # the wrapper maps [-bound, bound] back to [0,1]: feed both the same numbers
    tv_ref = ops.grad_total_variation((xb + 1) / 2, table, offsets, 0.5, lay.per_level_scale, 16, gridtype, False)
    t2 = table.cuda().requires_grad_()
    t2.grad = torch.zeros_like(t2)
    train_ops.grad_total_variation(t2, offsets.cuda(), lay.per_level_scale, 16, D, weight=0.5, inputs=xb.cuda(), bound=1, gridtype=gridtype)
    torch.cuda.synchronize()
    e_tv = (t2.grad.cpu() - tv_ref).abs().max().item() / max(1.0, tv_ref.abs().max().item())
    print(f"[D {D} gridtype {gridtype} interp {interp}, B {B}] dy_dx rel {e_dy:.2e}, input grad rel {e_gi:.2e} (bound {GRID_REL:.0e}); "
          f"table grad max |d| / S_e {tab_ratio:.2e} (bound {TABLE_REL:.1e} S_e + {TABLE_ABS:.0e}); adjoint rel {adj:.2e} (bound {ADJOINT_REL:.0e}); "
          f"TV rel {e_tv:.2e} (bound {TV_REL:.0e})")
    assert e_dy <= GRID_REL and e_gi <= GRID_REL
    assert tab_excess <= 0.0
    assert adj <= ADJOINT_REL
    assert e_tv <= TV_REL


# ------------------------------------------------------------------------------------------------ 6. the steady-state training step
def _train_model(sc):
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale = sc.density_scale
    m.conds = sc.cond
    return m.cuda().train()


def _gradient_mask(out, keep):
    """The field's outputs with their values unchanged and no gradient through the samples where keep is False."""
    return tuple(torch.where(keep.to(o.device).view(-1, *([1] * (o.dim() - 1))), o, o.detach()) for o in out)


def test_steady_state_training_step(monkeypatch):
    """mean_count at about 0.7 x the first step's sample count: a buffer of mean_count rounded up to 128 rows, rays past it composite
    to 0 / the background, every other ray and every gradient as in the oracle's render_train with the same mean_count.  Samples at a
    ReLU tie or an ambient cell face (found by the fp32 oracle) pass no gradient to the field in either implementation."""
    ops.build()
    torch.backends.cuda.matmul.allow_tf32 = False
    sc = scn.Scene(H=256, W=256, T=4, torso=False, density_scale=8.0)
    m = _train_model(sc)
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
    field_forward = ft.field_forward

    def oracle_field(p, hp, xyzs, dirs, cf, code, trace=None):
        if "mask" not in keep:
            tr = {}
            out = field_forward(p, hp, xyzs, dirs, cf, code, trace=tr)
            tie, face = ties(tr, out[2], hp, FLIP_BAND, CELL_BAND)
            keep["mask"] = ~(tie | face)
            keep["counts"] = (int(tie.sum()), int((face & ~tie).sum()))
        else:
            out = field_forward(p, hp, xyzs, dirs, cf, code)
        return _gradient_mask(out, keep["mask"])

    monkeypatch.setattr(ft, "field_forward", oracle_field)
    gpu_forward = m.forward
    monkeypatch.setattr(m, "forward", lambda *a, **k: _gradient_mask(gpu_forward(*a, **k), keep["mask"]))

    def oracle(dtype):
        p = ft.field_params(sc.state, dtype)
        emb = sc.state["individual_embeddings"].clone().to(dtype).requires_grad_(True)
        r = ft.render_train(p, sc.hparams, sc.state, fi["rays_o"], fi["rays_d"], cond_feat.to(dtype), emb[2], fi["bg_color"], sc.density_scale, 16,
                            mean_count=m.mean_count)
        ((r["rgb_map"].reshape(-1, 3).to(dtype) * coef_rgb.to(dtype)).sum() + (r["weights_sum"].to(dtype) * coef_ws.to(dtype)).sum() +
         (r["ambient"].to(dtype) * coef_amb.to(dtype)).sum()).backward()
        grads = {k: p[k].grad for k in ft.TRAINABLE}
        grads["code"] = emb.grad[2]
        return r, grads

    ref, r32 = oracle(torch.float32)
    _, r64 = oracle(torch.float64)
    m.zero_grad(set_to_none=True)
    res = m.render(*args, index=2, bg_color=fi["bg_color"].cuda(), perturb=False, max_steps=16)
    ((res["rgb_map"].reshape(-1, 3) * coef_rgb.cuda()).sum() + (res["weights_sum"] * coef_ws.cuda()).sum() + (res["ambient"] * coef_amb.cuda()).sum()).backward()
    torch.cuda.synchronize()
    assert m.step_counter[1].tolist() == [first, N] and res["position"].shape[0] == Mexp
    assert torch.equal(res["position"].detach().cpu(), ref["position"]), "samples differ from the oracle's"
    ro, rd = fi["rays_o"].reshape(-1, 3).contiguous(), fi["rays_d"].reshape(-1, 3).contiguous()
    nears, fars = ops.near_far_from_aabb(ro, rd, sc.state["aabb_train"], sc.hparams["min_near"])
    _, _, _, rays, _ = ops.march_rays_train(ro, rd, 1.0, sc.state["density_bitfield"], 1, sc.hparams["grid_size"], nears, fars, max_steps=16)
    over = (rays[:, 2] > 0) & (rays[:, 1] + rays[:, 2] > Mexp)
    bg = fi["bg_color"].reshape(-1, 3)
    ws, amb, rgb = res["weights_sum"].detach().cpu(), res["ambient"].detach().cpu(), res["rgb_map"].detach().cpu().reshape(-1, 3)
    assert float(ws[over].abs().max()) == 0.0 and float(amb[over].abs().max()) == 0.0 and torch.equal(rgb[over], bg[over].clamp(0, 1))
    e_out = {k: _rel(res[k].detach().cpu().reshape(-1), ref[k].detach().reshape(-1)) for k in ("rgb_map", "weights_sum", "ambient", "depth_map")}
    print(f"[steady step] first step {first} samples; mean_count {m.mean_count} -> M {Mexp}; {int(over.sum())} of {N} rays overflow; "
          f"{keep['counts'][0]} samples at a ReLU tie, {keep['counts'][1]} more at an ambient cell face; "
          "outputs rel " + ", ".join(f"{k} {v:.2e}" for k, v in e_out.items()) + f" (bound {FWD_REL:.0e})")
    assert max(e_out.values()) <= FWD_REL, e_out
    params = dict(m.named_parameters())
    got = {k: params[k].grad.cpu() for k in ft.TRAINABLE}
    got["code"] = params["individual_embeddings"].grad[2].cpu()
    _check_grads("[steady step]", got, r32, r64, cap=STEP_GRAD_CAP)


@pytest.mark.parametrize("steps", [3, 18])
def test_step_counter_and_mean_count(steps):
    """Each training render writes [its sample count, N] into step_counter row local_step % 16; update_extra_state then sets
    mean_count = int(sum of the first min(16, local_step) rows' counts / that number) and resets local_step (renderer.py:275-284)."""
    ops.build()
    sc = scn.Scene(H=64, W=64, T=steps, torso=False, density_scale=8.0)
    m = _train_model(sc)
    expect = torch.zeros(16, 2, dtype=torch.int64)
    counts = []
    for i in range(steps):
        fi = sc.frame_inputs(i)
        with torch.no_grad():
            m.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), None, None, index=0, bg_color=fi["bg_color"].cuda(), max_steps=16)
        ro, rd = fi["rays_o"].reshape(-1, 3).contiguous(), fi["rays_d"].reshape(-1, 3).contiguous()
        nears, fars = ops.near_far_from_aabb(ro, rd, sc.state["aabb_train"], sc.hparams["min_near"])
        _, _, _, _, c = ops.march_rays_train(ro, rd, 1.0, sc.state["density_bitfield"], 1, sc.hparams["grid_size"], nears, fars, max_steps=16)
        expect[i % 16] = torch.tensor([int(c[0]), int(c[1])])
        counts.append(int(c[0]))
    assert m.local_step == steps
    assert torch.equal(m.step_counter.cpu().long(), expect), (m.step_counter.cpu(), expect)
    noise = (scn.hashed_uniform(128 ** 3 * 3, 7, 1.0) + 0.5).view(1, 128, 128, 128, 3)
    m.update_extra_state(cond_index=0, noise=noise)
    total = min(16, steps)
    want = int(expect[:total, 0].sum().item() / total)
    print(f"[{steps} steps] counts {counts}; mean_count {m.mean_count} (formula {want})")
    assert m.mean_count == want and m.local_step == 0
    assert len(set(counts)) > 1
