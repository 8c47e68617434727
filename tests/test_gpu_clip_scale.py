"""The fused renderer at clip scale: calls that hold many frames, frames with different round schedules, every precision mode.

bench.py times gfpp_render_frames with 50 frames per call at 512x512 (render_clip's default is 64 frames per call); the parity tests
render one or two frames per call.  Several code paths only switch on when a call holds many frames, or frames that differ: the
frame index taken from hit records and survivor ids, k_head_v2's per-frame conditioning images, the per-frame death histograms,
sample counts and pass-2 caps (k_schedule), the epilogue's per-frame torso biases and pixel counts, k_ray_setup warps that straddle
two frames (N not a multiple of 32), hit lists past 2^31 bytes and the render workspace a model reuses across calls of other shapes.

  * Every ray gets the same arithmetic wherever it is scheduled (MMAs are independent per row, each ray is composited sequentially
    by its owner thread; DESIGN.md section 5), so a frame of a multi-frame call must be BIT-IDENTICAL (torch.equal) to the same frame
    rendered alone -- every map and every per-frame statistic, in all five precisions (k_head: fp32; k_head_v2: fp16, robust;
    k_head_tc: bf16x3, bf16).
  * Against the fp32 CPU oracle the bars of test_gpu_render.py / test_gpu_v2.py: 5e-6 max-abs for fp32, 1e-3 and PSNR >= 50 dB for
    the tensor-core modes, knife-edge rays excluded from the max-abs bar and counted; the round-schedule cap B and the torso pixel
    count P exact, the valid-sample count S within the knife-edge count."""
import functools

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from helpers import build_model, lively_state, parity_report

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16", "robust", "bf16x3", "bf16"]
KERNEL = {"fp32": "k_head", "fp16": "k_head_v2", "robust": "k_head_v2", "bf16x3": "k_head_tc", "bf16": "k_head_tc"}
PSNR_MIN = 50.0
MAPS = ("rgb_map", "depth_map", "weights_sum", "torso_alpha_map", "torso_rgb_map", "deform")
PER_FRAME = ("poses_c2w", "pose6", "rays_o", "rays_d")    # render_frames arguments with a leading frame axis


def _tol(precision):
    return 5e-6 if precision == "fp32" else 1e-3


@functools.lru_cache(maxsize=None)
def _scene(H, W, T, torso, max_steps, ds):
    return scn.Scene(H=H, W=W, T=T, torso=torso, max_steps=max_steps, density_scale=ds)


def _model(sc, precision, state=None):
    return build_model(sc, state, precision=precision)


def _same(a, b):
    """torch.equal, with NaN positions (the depth of rays that miss the aabb) required to match as well."""
    if not a.is_floating_point():
        return torch.equal(a, b)
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0), b.masked_fill(nb, 0.0))


def _rays(sc, frames, moved=None):
    """get_rays of `frames` as [F,N,3] pairs; moved[i] (bool [N]): rays of frame i shifted off the volume (rays_o.y += 6, as
    test_gpu_render.py::test_rays_missing_the_volume)."""
    ro = torch.cat([sc.frame_inputs(t)["rays_o"] for t in frames])
    rd = torch.cat([sc.frame_inputs(t)["rays_d"] for t in frames])
    if moved is not None:
        for i, m in enumerate(moved):
            ro[i, m, 1] += 6.0
    return ro, rd


def _kwargs(sc, frames, rays=None, max_steps=None):
    """render_frames keyword arguments for `frames` of `sc`: rays generated in-kernel from the poses, or the given [F,N,3] rays."""
    poses = torch.stack([sc.pose(t) for t in frames])
    kw = dict(pose6=scn.convert_poses(poses).cuda() if sc.torso else None, bg_coords=sc.bg_coords.cuda() if sc.torso else None,
              bg_color=sc.bg_color.cuda(), dt_gamma=sc.hparams["dt_gamma"],
              max_steps=sc.hparams["max_steps"] if max_steps is None else max_steps, T_thresh=sc.T_thresh)
    if rays is None:
        kw.update(poses_c2w=poses.cuda(), intrinsics=sc.intrinsics, H=sc.H, W=sc.W)
    else:
        kw.update(rays_o=rays[0].cuda(), rays_d=rays[1].cuda())
    return kw


def _one(kw, f):
    return {k: (v[f:f + 1] if k in PER_FRAME and v is not None else v) for k, v in kw.items()}


def _clip_feat(model, sc, frames):
    return model.cal_cond_feat_clip(sc.cond.cuda())[list(frames)]


def _frame_feat(model, sc, frames):
    """The conditioning render() computes for each frame (cal_cond_feat of its window), as the oracle does."""
    return torch.stack([model.cal_cond_feat(sc.frame_inputs(t)["cond"].cuda()).reshape(-1) for t in frames])


def _split_check(model, feat, kw, label):
    """One call of F frames against F calls of one frame: every map bit-identical, per-frame B, S and P equal, and the call's
    survivor count equal to the sum of the single-frame ones.  Returns the call's result and the single-frame stats [F,4] (CPU)."""
    Fn = feat.shape[0]
    full = model.render_frames(feat, want_stats=True, **kw)
    keys = [k for k in MAPS if k in full]
    st = full["stats"].cpu()
    bad, singles = [], []
    for f in range(Fn):
        one = model.render_frames(feat[f:f + 1], want_stats=True, **_one(kw, f))
        bad += [(f, k) for k in keys if not _same(full[k][f], one[k][0])]
        singles.append(one["stats"][0].cpu())
    singles = torch.stack(singles)
    stats_bad = [f for f in range(Fn) if not torch.equal(st[f, [0, 2, 3]], singles[f, [0, 2, 3]])]
    print(f"[{label}] F={Fn}: frames with every map ({', '.join(keys)}) bit-identical to the single-frame call {Fn - len({f for f, _ in bad})} "
          f"of {Fn} (bound {Fn}); per-frame (B, S, P) equal {Fn - len(stats_bad)} of {Fn}; B values {sorted(set(st[:, 0].tolist()))}; "
          f"survivors {int(st[0, 1])} vs sum of single-frame calls {int(singles[:, 1].sum())}")
    assert not bad, f"maps that differ from the single-frame call (frame, map): {bad[:12]}"
    assert not stats_bad, [(f, st[f].tolist(), singles[f].tolist()) for f in stats_bad[:8]]
    assert int(st[0, 1]) == int(singles[:, 1].sum())
    return full, singles


# ------------------------------------------------------------------------------------------------ 1. many frames per call
SPLIT_SHAPES = {
    # name: (H, W, F, in-kernel rays, max_steps, density_scale)
    "bench512_F50": (512, 512, 50, True, 16, 8.0),       # what bench.py times: 50 frames per call, rays from the poses
    "ragged50_F37": (50, 50, 37, False, 8, 1.0),         # N = 2 500: warps and tiles straddle frames; translucent, so pass 2 runs
}


@pytest.mark.parametrize("shape", list(SPLIT_SHAPES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_multi_frame_call_equals_single_frame_calls(precision, shape):
    H, W, Fn, in_kernel, ms, ds = SPLIT_SHAPES[shape]
    sc = _scene(H, W, Fn, True, ms, ds)
    model = _model(sc, precision)
    frames = list(range(Fn))
    kw = _kwargs(sc, frames, None if in_kernel else _rays(sc, frames))
    _, singles = _split_check(model, _clip_feat(model, sc, frames), kw, f"{shape} {precision}/{KERNEL[precision]}")
    if shape.startswith("ragged"):
        assert int(singles[:, 1].min()) > 0, "every frame must have rays that reach pass 2"


@pytest.mark.parametrize("precision", ["fp16", "robust"])
def test_render_clip_default_chunking_equals_single_frame_calls(precision):
    """render_clip's default frames_per_call = 64 on a 150-frame clip: calls of 64, 64 and 22 frames, fp32 frames and uint8 frames
    written into a preallocated buffer, against the stacked single-frame results."""
    T = 150
    sc = _scene(512, 512, T, True, 16, 8.0)
    model = _model(sc, precision)
    frames = list(range(T))
    feat = _clip_feat(model, sc, frames)
    poses = torch.stack([sc.pose(t) for t in frames])
    ckw = dict(cond_feat=feat, bg_color=sc.bg_color, bg_coords=sc.bg_coords, T_thresh=sc.T_thresh)
    rgb = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, **ckw)
    u8 = torch.empty(T, sc.H * sc.W, 3, dtype=torch.uint8, device="cuda")
    ret = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, out=u8, as_uint8=True, **ckw)
    assert ret.data_ptr() == u8.data_ptr()
    kw = _kwargs(sc, frames)
    bad = []
    for f in range(T):
        one = model.render_frames(feat[f:f + 1], want_aux=False, want_torso_maps=False, **_one(kw, f))["rgb_map"][0]
        if not torch.equal(rgb[f], one):
            bad.append(f)
    u8_ok = torch.equal(u8.int(), (rgb * 255.0).int())
    print(f"[render_clip T={T} frames_per_call=64 {precision}] fp32 frames bit-identical to single-frame calls {T - len(bad)} of {T} "
          f"(bound {T}); uint8 frames == (rgb*255).int(): {u8_ok}")
    assert not bad, bad[:12]
    assert u8_ok


# ------------------------------------------------------------------------------------------------ 2. frames with different schedules
# frame f moves MOVED[f] of its rays off the volume (a scrambled 1/1000 pattern of the ray index).  On the 64x64 translucent scene
# (density_scale 1, max_steps 8) the oracle's schedules give B = 9, 10, 9, 12, 8, 9, 9, 1: the clamp N // n_alive takes the values
# 2, 3, 4, 5..6, 7, 8, 8 after the first round, and the last frame has no ray left after it.
MOVED = [0.0, 0.3, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0]


def _moved_mask(N, frac):
    return (torch.arange(N) * 7919) % 1000 < round(1000 * frac)


def _oracle(sc, state, t, rays, torso=None):
    from oracle.render import OracleModel
    fi = sc.frame_inputs(t)
    orc = OracleModel(state, sc.hparams, torso=torso)
    orc.density_scale = sc.density_scale
    return orc.render(rays[0].reshape(1, -1, 3), rays[1].reshape(1, -1, 3), fi["cond"], fi["bg_coords"], fi["poses"],
                      bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **sc.hparams)


def _b_comparable(ref, max_steps):
    """test_gpu_render.py::test_render_matches_oracle's rule: B is compared when the oracle's loop ran to max_steps with rays alive."""
    sched = ref["stats"]["schedule"]
    return sched[-1][0] > 0 and sum(s for _, s in sched) >= max_steps


def _oracle_check(label, precision, ref, rgb, stats, ms, ws=None, tol=None, knife_tol=1e-3):
    """rgb (and weights_sum) of one frame against the oracle; B (under _b_comparable) and P exact, S within the knife-edge count."""
    tol = _tol(precision) if tol is None else tol
    rep = parity_report(rgb.reshape(-1, 3), ref["rgb_map"].reshape(-1, 3), ref["knife"], knife_tol=knife_tol)
    repw = parity_report(ws.reshape(-1), ref["weights_sum"].reshape(-1), ref["knife"], knife_tol=knife_tol) if ws is not None else None
    B, S, P = int(stats[0]), int(stats[2]), int(stats[3])
    rs = ref["stats"]
    print(f"[{label} {precision}] rgb max|d|={rep['max_abs']:.2e} (bound {tol:.0e}; all {rep['max_abs_all']:.2e}, knife-edge rays "
          f"{rep['n_knife']}) psnr={rep['psnr']:.1f} dB (bound {PSNR_MIN:.0f})"
          + (f" | alpha max|d|={repw['max_abs']:.2e}" if repw else "")
          + f" | B={B} (oracle {rs['B_total']}{'' if _b_comparable(ref, ms) else ', not compared'}) P={P} ({rs['P']}) "
          f"S={S} ({rs['S']}, bound +-{rep['n_knife']})")
    assert rep["max_abs"] <= tol and rep["psnr"] >= PSNR_MIN, (label, precision, rep)
    if repw is not None:
        assert repw["max_abs"] <= tol, (label, precision, repw)
    if _b_comparable(ref, ms):
        assert B == rs["B_total"], (label, B, rs["B_total"])
    assert P == rs["P"], (label, P, rs["P"])
    assert abs(S - rs["S"]) <= rep["n_knife"], (label, S, rs["S"], rep["n_knife"])


@pytest.fixture(scope="module")
def schedules(oracle_ops):
    """The 8-frame call of part 2: rays with MOVED fractions off the volume, the oracle's frames, and a 3-frame call of rays that all miss."""
    sc = _scene(64, 64, 8, True, 8, 1.0)
    N = sc.H * sc.W
    frames = list(range(8))
    rays = _rays(sc, frames, [_moved_mask(N, f) for f in MOVED])
    refs = [_oracle(sc, sc.state, t, (rays[0][t], rays[1][t])) for t in frames]
    head = _scene(64, 64, 8, False, 8, 1.0)
    miss = _rays(head, [0, 1, 2], [torch.ones(N, dtype=torch.bool)] * 3)
    miss_refs = [_oracle(head, head.state, t, (miss[0][t], miss[1][t])) for t in range(3)]
    return sc, frames, rays, refs, head, miss, miss_refs


@pytest.mark.parametrize("precision", PRECISIONS)
def test_frames_with_different_round_schedules(schedules, precision):
    sc, frames, rays, refs, _, _, _ = schedules
    ms = sc.hparams["max_steps"]
    model = _model(sc, precision)
    feat = _frame_feat(model, sc, frames)
    kw = _kwargs(sc, frames, rays)
    # the premise, from the oracle's schedules and the single-frame stats: B differs between frames and pass 2 has work in several
    Bs = [r["stats"]["B_total"] for r in refs]
    single = torch.stack([model.render_frames(feat[f:f + 1], want_stats=True, **_one(kw, f))["stats"][0].cpu() for f in frames])
    n_pass2 = int((single[:, 1] > 0).sum())
    print(f"[schedules {precision}] oracle B per frame {Bs} ({len(set(Bs))} distinct, bound >= 4); pass-2 survivors per frame "
          f"{single[:, 1].tolist()} ({n_pass2} frames, bound >= 3)")
    assert len(set(Bs)) >= 4 and n_pass2 >= 3
    res, _ = _split_check(model, feat, kw, f"schedules {precision}/{KERNEL[precision]}")
    st = res["stats"].cpu()
    for f in frames:
        _oracle_check(f"schedules f{f} moved {MOVED[f]:.1f}", precision, refs[f], res["rgb_map"][f].cpu(), st[f], ms,
                      ws=res["weights_sum"][f].cpu())


@pytest.mark.parametrize("precision", PRECISIONS)
def test_call_where_every_ray_misses(schedules, precision):
    """n_hits = 0: both passes of the head kernel start with an empty list.  The head model, so that the image is exactly the
    background (with a torso the background goes through the torso MLP, whose fp32 sums are not the oracle's bit for bit)."""
    _, _, _, _, head, miss, miss_refs = schedules
    model = _model(head, precision)
    feat = _frame_feat(model, head, [0, 1, 2])
    res = model.render_frames(feat, want_stats=True, **_kwargs(head, [0, 1, 2], miss))
    st = res["stats"].cpu()
    eq = [torch.equal(res["rgb_map"][f].cpu(), miss_refs[f]["rgb_map"].reshape(-1, 3)) for f in range(3)]
    print(f"[all rays miss, 3 frames, {precision}/{KERNEL[precision]}] rgb == oracle {eq}; depth all NaN "
          f"{bool(torch.isnan(res['depth_map']).all())}; weights_sum max {res['weights_sum'].max().item()}; B {st[:, 0].tolist()} (bound 1); "
          f"S {st[:, 2].tolist()}; survivors {int(st[0, 1])}")
    assert all(eq)
    assert torch.isnan(res["depth_map"]).all() and all(torch.isnan(r["depth_map"]).all() for r in miss_refs)
    assert (res["weights_sum"] == 0).all()
    assert st[:, 0].tolist() == [1, 1, 1] and all(r["stats"]["B_total"] == 1 for r in miss_refs)
    assert st[:, 2].tolist() == [0, 0, 0] and int(st[0, 1]) == 0


# ------------------------------------------------------------------------------------------------ 3. the benchmarked call vs the oracle
BENCH_CHECKED = [0, 25, 49]
LIVELY_CHECKED = [0, 15]


@pytest.fixture(scope="module")
def bench_oracle(oracle_ops):
    """The oracle's frames 0, 25 and 49 of the 512x512 bench clip on the rays the kernel generates (fp32, shared by all modes)."""
    sc = _scene(512, 512, 50, True, 16, 8.0)
    m = _model(sc, "fp32")
    ro, rd = m.generate_rays(torch.stack([sc.pose(t) for t in BENCH_CHECKED]), sc.intrinsics, sc.H, sc.W)
    refs = {t: _oracle(sc, sc.state, t, (ro[i].cpu(), rd[i].cpu())) for i, t in enumerate(BENCH_CHECKED)}
    return sc, refs


@pytest.mark.parametrize("precision", PRECISIONS)
def test_benchmarked_call_vs_oracle(bench_oracle, precision):
    """render_clip(frames_per_call=50) at 512x512, rays generated in-kernel: one call of the 50 frames bench.py times."""
    sc, refs = bench_oracle
    model = _model(sc, precision)
    frames = list(range(50))
    poses = torch.stack([sc.pose(t) for t in frames])
    rgb, stats = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=_clip_feat(model, sc, frames), bg_color=sc.bg_color,
                                   bg_coords=sc.bg_coords, T_thresh=sc.T_thresh, frames_per_call=50, want_stats=True)
    st = stats.cpu()
    for t in BENCH_CHECKED:
        _oracle_check(f"bench 512 F=50 f{t}", precision, refs[t], rgb[t].cpu(), st[t], sc.hparams["max_steps"])


@pytest.fixture(scope="module")
def lively_oracle(oracle_ops):
    """The lively scene (gain 4, table decay 1; colours and densities with O(1) range) at 96x96: oracle frames 0 and 15 on the
    kernel's rays.  density_scale 1: at 16 the robust mode is at the edge of 1e-3 on single frames already (DESIGN.md section 6;
    1.4e-3 at frame 0 of this 96x96 scene, through render() and get_rays' rays as well)."""
    sc = scn.Scene(H=96, W=96, T=16, torso=False, density_scale=1.0, table_decay=1.0, table_amp=1.0)
    state = lively_state(sc.state, 4.0)
    m = _model(sc, "fp32", state)
    ro, rd = m.generate_rays(torch.stack([sc.pose(t) for t in LIVELY_CHECKED]), sc.intrinsics, sc.H, sc.W)
    refs = {t: _oracle(sc, state, t, (ro[i].cpu(), rd[i].cpu())) for i, t in enumerate(LIVELY_CHECKED)}
    return sc, state, refs


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "robust"])
def test_lively_scene_clip_vs_oracle(lively_oracle, precision):
    """The modes that hold 1e-3 on the lively scene (test_gpu_render_tc.py, test_gpu_v2.py), in one 16-frame call; rays within 3 %
    of the termination threshold count as knife-edge there too."""
    sc, state, refs = lively_oracle
    model = _model(sc, precision, state)
    frames = list(range(16))
    poses = torch.stack([sc.pose(t) for t in frames])
    feat = _clip_feat(model, sc, frames)
    rgb, stats = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=feat, bg_color=sc.bg_color, T_thresh=sc.T_thresh,
                                   frames_per_call=16, want_stats=True)
    st = stats.cpu()
    for t in LIVELY_CHECKED:
        one = model.render_clip(poses[t:t + 1], sc.intrinsics, sc.H, sc.W, cond_feat=feat[t:t + 1], bg_color=sc.bg_color,
                                T_thresh=sc.T_thresh, frames_per_call=1)
        assert torch.equal(rgb[t], one[0]), f"frame {t} of the 16-frame call differs from its single-frame call"
        _oracle_check(f"lively 96 F=16 f{t}", precision, refs[t], rgb[t].cpu(), st[t], sc.hparams["max_steps"], tol=1e-3, knife_tol=3e-2)


# ------------------------------------------------------------------------------------------------ 4. a hit list past 2^31 bytes
def test_hit_list_past_2gb():
    """160 frames of 512x512 with the focal length tripled (the head fills the frame): ~42 M rays, > 2^25 of them with a 64-byte hit
    record, so records sit past byte 2^31 of the list.  Which frames land there depends on arrival order: every frame is compared.
    Peak device memory ~5 GB (workspace 92 B per ray plus the outputs); released at the end."""
    sc = _scene(512, 512, 160, False, 16, 8.0)
    fx, fy, cx, cy = sc.intrinsics
    intr = (3 * fx, 3 * fy, cx, cy)
    Fn = 160
    frames = list(range(Fn))
    model = _model(sc, "fp16")
    feat = _clip_feat(model, sc, frames)
    poses = torch.stack([sc.pose(t) for t in frames]).cuda()
    kw = dict(intrinsics=intr, H=sc.H, W=sc.W, bg_color=sc.bg_color.cuda(), dt_gamma=sc.hparams["dt_gamma"],
              max_steps=sc.hparams["max_steps"], T_thresh=sc.T_thresh)
    try:
        for precision in ("fp16", "bf16x3", "fp32"):
            model.mlp_precision = precision
            full = model.render_frames(feat, poses_c2w=poses, **kw)
            n_hit = int((full["weights_sum"] > 0).sum())
            bad = []
            for f in frames:
                one = model.render_frames(feat[f:f + 1], poses_c2w=poses[f:f + 1], **kw)
                if not (torch.equal(full["rgb_map"][f], one["rgb_map"][0]) and torch.equal(full["weights_sum"][f], one["weights_sum"][0])):
                    bad.append(f)
            print(f"[hit list {precision}/{KERNEL[precision]}] F={Fn} x 512^2 = {Fn * sc.H * sc.W} rays; rays with weights_sum > 0: "
                  f"{n_hit} (bound > 2^25 = {2 ** 25}), hit list >= {64 * n_hit / 2 ** 30:.2f} GiB; frames bit-identical to the "
                  f"single-frame call {Fn - len(bad)} of {Fn} (bound {Fn}); workspace {model._workspace.numel() / 2 ** 30:.2f} GiB")
            assert n_hit > 2 ** 25
            assert not bad, bad[:12]
            del full, one
    finally:
        model._workspace = None
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ 5. workspace reuse
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_workspace_reuse_across_call_shapes(precision):
    """One model renders calls of different F, N, max_steps and density_scale in turn, reusing its workspace (only the histogram ..
    pixel-count range is zeroed per call); each result equals the same call on a fresh model."""
    big = _scene(512, 512, 50, True, 16, 8.0)
    ragged = _scene(50, 50, 3, True, 1024, 1.0)
    small = _scene(64, 64, 1, True, 8, 8.0)
    calls = [("512^2 F=50 max_steps 16", big, list(range(50)), False),
             ("50x50 F=3 max_steps 1024 ds 1", ragged, [0, 1, 2], True),
             ("64^2 F=1 max_steps 8", small, [0], False)]
    calls.append(calls[0])

    def run(model, sc, frames, supplied):
        model.density_scale = sc.density_scale
        kw = _kwargs(sc, frames, _rays(sc, frames) if supplied else None)
        return model.render_frames(_clip_feat(model, sc, frames), want_stats=True, **kw)

    reused = _model(big, precision)
    fresh = {}
    for i, (label, sc, frames, supplied) in enumerate(calls):
        got = run(reused, sc, frames, supplied)
        if label not in fresh:
            fresh[label] = run(_model(sc, precision), sc, frames, supplied)
        ref = fresh[label]
        bad = [k for k in list(MAPS) + ["stats"] if k in ref and not _same(got[k], ref[k])]
        print(f"[workspace reuse {precision}, call {i + 1}: {label}] outputs that differ from a fresh model's: {bad} (bound none); "
              f"workspace {reused._workspace.numel() / 2 ** 20:.0f} MiB")
        assert not bad, (label, bad)


# ------------------------------------------------------------------------------------------------ 6. torso-SR composite, several frames
def test_torso_sr_composite_multi_frame():
    """gfpp_torso_sr_composite with F = 8 (RADNeRFTorsowithSR.render_clip's chunk) against 8 one-frame calls, each frame with its own
    head image, weights_sum and lm68 row: bit for bit, per-frame torso pixel counts included."""
    import json
    import os
    from genefaceplusplus_b200.config import may_hparams
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "torso_sr256.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    hp = may_hparams(**{**meta["overrides"], "torso_head_aware": True})
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m = m.cuda().eval()
    sc = _scene(256, 256, 8, True, 16, 8.0)
    Fn, N = 8, 256 * 256
    g = torch.Generator().manual_seed(8)
    ws = torch.rand(Fn, N, generator=g)
    image = torch.rand(Fn, N, 3, generator=g) * ws.unsqueeze(-1)
    lm68 = scn.lm68_sequence(Fn)
    bg_coords, bg_color = sc.bg_coords.cuda(), sc.bg_color.cuda()
    full = m.torso_composite_native(image.cuda(), ws.cuda(), lm68.cuda(), bg_coords, bg_color)
    keys = ("rgb_map", "torso_alpha_map", "torso_rgb_map", "deform", "torso_pixels")
    bad = []
    for f in range(Fn):
        one = m.torso_composite_native(image[f:f + 1].cuda(), ws[f:f + 1].cuda(), lm68[f:f + 1].cuda(), bg_coords, bg_color)
        bad += [(f, k) for k in keys if not torch.equal(full[k][f], one[k][0])]
    px = full["torso_pixels"].tolist()
    print(f"[torso-SR composite F={Fn} 256^2] maps and torso pixel counts that differ from one-frame calls: {bad} (bound none); "
          f"torso pixels per frame {px}")
    assert not bad
    assert min(px) > 0
