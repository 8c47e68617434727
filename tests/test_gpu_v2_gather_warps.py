"""The gather warps of the fp16 row-owner head kernel (k_head_v2<false>, DESIGN §5): one producer warp per slot looks up the
position-grid levels of every row's next sample and hands them to the row owners through a per-row staging slot, with a
request / reply pair of mbarriers per slot and a final request that releases the warp when the owners leave.

The hand-off must not change a bit: a row's features come from the same per-level arithmetic (gather8.cuh) whichever warp computes
them, and a frame's rays get the same arithmetic wherever they are scheduled (DESIGN §5).  So every frame of a multi-frame call is
compared with torch.equal against the same frame rendered by a one-frame call, on the shapes where the protocol meets its edge
cases: the bench's 50-frame 512^2 call, CTAs with fewer rays than rows (64^2, one frame), pass 2 (50x50, max_steps 8, translucent),
a call whose rays all miss (no batch holds a live row; the gather warps still serve the prologue's request and must be released),
and jittered ray starts.  Where the existing tests compare with the fp32 CPU oracle (one 64^2 frame, the all-miss call), so does this
file, with the same bars."""
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from helpers import build_model, parity_report

pytestmark = pytest.mark.gpu
PER_FRAME = ("poses_c2w", "pose6", "rays_o", "rays_d", "noise")
MAPS = ("rgb_map", "depth_map", "weights_sum", "torso_alpha_map", "torso_rgb_map", "deform")


def _same(a, b):
    """torch.equal, NaN positions (the depth of rays that miss the aabb) included."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0), b.masked_fill(nb, 0.0))


def _kwargs(sc, frames, max_steps=None, rays=None, noise=None):
    poses = torch.stack([sc.pose(t) for t in frames])
    kw = dict(pose6=scn.convert_poses(poses).cuda() if sc.torso else None, bg_coords=sc.bg_coords.cuda() if sc.torso else None,
              bg_color=sc.bg_color.cuda(), dt_gamma=sc.hparams["dt_gamma"],
              max_steps=sc.hparams["max_steps"] if max_steps is None else max_steps, T_thresh=sc.T_thresh, noise=noise)
    if rays is None:
        kw.update(poses_c2w=poses.cuda(), intrinsics=sc.intrinsics, H=sc.H, W=sc.W)
    else:
        kw.update(rays_o=rays[0].cuda(), rays_d=rays[1].cuda())
    return kw


def _frame_rays(sc, frames, off_volume=False):
    ro = torch.cat([sc.frame_inputs(t)["rays_o"] for t in frames])
    rd = torch.cat([sc.frame_inputs(t)["rays_d"] for t in frames])
    if off_volume:   # as test_gpu_render.py::test_rays_missing_the_volume
        ro[..., 1] += 6.0
    return ro, rd


def _against_single_frame_calls(sc, frames, label, **kwargs):
    """One fp16 call of `frames`, then each frame alone (stored): every map and B / S / P bit-identical.  Returns the call's result."""
    model = build_model(sc, precision="fp16")
    feat = model.cal_cond_feat_clip(sc.cond.cuda())[list(frames)]
    kw = _kwargs(sc, frames, **kwargs)
    singles = [model.render_frames(feat[f:f + 1], want_stats=True, **{k: (v[f:f + 1] if k in PER_FRAME and v is not None else v)
                                                                      for k, v in kw.items()}) for f in range(len(frames))]
    full = model.render_frames(feat, want_stats=True, **kw)
    keys = [k for k in MAPS if k in full]
    bad = [(f, k) for f, one in enumerate(singles) for k in keys if not _same(full[k][f], one[k][0])]
    st = full["stats"].cpu()
    st_bad = [f for f, one in enumerate(singles) if not torch.equal(st[f, [0, 2, 3]], one["stats"][0, [0, 2, 3]].cpu())]
    survivors = sum(int(one["stats"][0, 1]) for one in singles)
    print(f"[gather warps, {label}] F={len(frames)}: maps differing from the single-frame calls {bad[:8]}; (B, S, P) differing {st_bad[:8]}; "
          f"survivors {int(st[0, 1])} vs {survivors}")
    assert not bad and not st_bad
    assert int(st[0, 1]) == survivors
    return full


def _oracle(sc, t, rays):
    from oracle.render import OracleModel
    orc = OracleModel(sc.state, sc.hparams)
    orc.density_scale = sc.density_scale
    fi = sc.frame_inputs(t)
    return orc.render(rays[0].view(1, -1, 3), rays[1].view(1, -1, 3), fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"],
                      T_thresh=sc.T_thresh, **sc.hparams)


def test_one_frame_64_matches_oracle(oracle_ops):
    # 4 096 rays over every SM: most CTAs' slots hold no live row in any batch
    sc = scn.Scene(H=64, W=64, T=2, torso=True, density_scale=8.0)
    model = build_model(sc, precision="fp16")
    feat = model.cal_cond_feat_clip(sc.cond.cuda())[[1]]
    kw = _kwargs(sc, [1])
    a = model.render_frames(feat, want_stats=True, **kw)
    b = model.render_frames(feat, want_stats=True, **kw)
    rays = model.generate_rays(sc.pose(1).view(1, 4, 4).cuda(), sc.intrinsics, 64, 64)
    ref = _oracle(sc, 1, (rays[0][0].cpu(), rays[1][0].cpu()))
    rep = parity_report(a["rgb_map"][0].cpu(), ref["rgb_map"].view(-1, 3), ref["knife"])
    print(f"[gather warps, 64^2 F=1] rgb max|d| vs oracle {rep['max_abs']:.2e} (knife {rep['n_knife']}), psnr {rep['psnr']:.1f}")
    assert all(_same(a[k], b[k]) for k in MAPS if k in a), "two identical calls must render identical frames"
    assert rep["max_abs"] <= 1e-3 and rep["psnr"] >= 50


def test_bench_call_512_50_frames():
    sc = scn.Scene(H=512, W=512, T=50, torso=True, density_scale=8.0)
    _against_single_frame_calls(sc, list(range(50)), "512^2 F=50")


def test_pass2_50x50_max_steps_8():
    sc = scn.Scene(H=50, W=50, T=50, torso=True, max_steps=8, density_scale=1.0)
    frames = list(range(50))
    full = _against_single_frame_calls(sc, frames, "50x50 F=50 max_steps 8", rays=_frame_rays(sc, frames))
    assert int(full["stats"][0, 1]) > 0, "rays must reach pass 2"


def test_every_ray_misses(oracle_ops):
    # head model, as test_gpu_clip_scale.py::test_call_where_every_ray_misses: the frame is the background, exactly the oracle's
    sc = scn.Scene(H=64, W=64, T=3, torso=False, density_scale=8.0)
    frames = [0, 1, 2]
    rays = _frame_rays(sc, frames, off_volume=True)
    full = _against_single_frame_calls(sc, frames, "all rays miss", rays=rays)
    assert float(full["weights_sum"].abs().max()) == 0.0 and torch.isnan(full["depth_map"]).all()
    for f in frames:
        ref = _oracle(sc, f, (rays[0][f], rays[1][f]))
        assert torch.equal(full["rgb_map"][f].cpu(), ref["rgb_map"].reshape(-1, 3))


def test_perturb():
    sc = scn.Scene(H=64, W=64, T=4, torso=True, density_scale=8.0)
    frames = [0, 1, 2, 3]
    noise = torch.rand(len(frames), 64 * 64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(11))
    full = _against_single_frame_calls(sc, frames, "perturb", noise=noise)
    model = build_model(sc, precision="fp16")
    plain = model.render_frames(model.cal_cond_feat_clip(sc.cond.cuda())[frames], **_kwargs(sc, frames))
    assert not torch.equal(full["rgb_map"], plain["rgb_map"]), "the jitter must move the samples"
