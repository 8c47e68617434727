"""Alpha-matte frames of the fused renderer on the GPU: k_epilogue's coverage `alpha_map` and premultiplied RGBA `rgba_u8`
(include/gfpp.h, gfpp_outputs), on the golden scenes and the 512x512 bench scene, in all five mlp_precision modes.

  * Coverage: alpha_map is ws + (1 - ws) * torso_alpha recomputed in fp32 from the same call's weights_sum and torso_alpha_map, bit for
    bit (head-only models: weights_sum itself); against the reference's CPU render (tests/golden) within the 1e-3 bar of
    test_gpu_render.py, knife-edge rays excluded as there.
  * Compositing: P + (1 - A) * B, with P the fp32 frame over a zero background, matches the frame rendered over a random background B
    to 2e-6 wherever that frame is not clamped.
  * uint8: the colour bytes of rgba_u8 are rgb_u8 over a zero background, the fourth byte is (uint8)(int)(alpha_map * 255); an
    rgba_u8-only call writes the same bytes.
  * Nothing else moves: every other output and the stats are bit-identical with and without the matte outputs.
  * Clip scale: a 50-frame render_clip(as_rgba=True) equals its frames_per_call=7 rendering; iter_video_frames(as_rgba=True) yields
    exactly render_driver_batch(as_rgba=True)."""
import functools
import glob
import json
import os
import re

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import driver
from genefaceplusplus_b200 import scene as scn
from helpers import build_model, parity_report

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16", "robust", "bf16x3", "bf16"]
GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")) if re.match(r"(head|torso)\d+_ms", os.path.basename(p)))
CASES = [os.path.basename(p)[:-4] for p in GOLDEN] + ["bench512"]
OTHER = ("rgb_map", "rgb_u8", "weights_sum", "depth_map", "torso_alpha_map", "torso_rgb_map", "deform", "stats")
TOL_ORACLE = 1e-3
TOL_COMPOSITE = 2e-6


@functools.lru_cache(maxsize=None)
def _case(name):
    """(scene, frames, T_thresh, golden arrays or None)"""
    if name == "bench512":
        sc = scn.Scene(H=512, W=512, T=8, torso=True, density_scale=8.0)
        return sc, [0, 3, 7], sc.T_thresh, None
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
    m = json.loads(bytes(z["meta"]).decode())
    sc = scn.Scene(H=m["size"], W=m["size"], T=8, torso=m["torso"], max_steps=m["max_steps"], density_scale=m["density_scale"])
    return sc, m["frames"], m["T_thresh"], z


def _same(a, b):
    """torch.equal with NaN positions (the depth of rays that miss the volume) required to match."""
    if not a.is_floating_point():
        return torch.equal(a, b)
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0), b.masked_fill(nb, 0.0))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", CASES)
def test_matte(name, precision):
    sc, frames, T_thresh, gold = _case(name)
    model = build_model(sc, precision=precision)
    fis = [sc.frame_inputs(t) for t in frames]
    feat = torch.stack([model.cal_cond_feat(fi["cond"].cuda()).reshape(-1) for fi in fis])
    kw = dict(rays_o=torch.cat([fi["rays_o"] for fi in fis]).cuda(), rays_d=torch.cat([fi["rays_d"] for fi in fis]).cuda(),
              dt_gamma=sc.hparams["dt_gamma"], max_steps=sc.hparams["max_steps"], T_thresh=T_thresh)
    if sc.torso:
        kw.update(pose6=torch.cat([fi["poses"] for fi in fis]).cuda(), bg_coords=sc.bg_coords.cuda())
    Fn, N = len(frames), sc.H * sc.W
    B = torch.rand(N, 3, generator=torch.Generator().manual_seed(11))

    def call(bg, matte):
        bufs = dict(rgb_out=torch.empty(Fn, N, 3, device="cuda"), u8_out=torch.empty(Fn, N, 3, dtype=torch.uint8, device="cuda"))
        if matte:
            bufs.update(alpha_out=torch.empty(Fn, N, device="cuda"), rgba_out=torch.empty(Fn, N, 4, dtype=torch.uint8, device="cuda"))
        r = model.render_frames(feat, bg_color=bg.cuda(), want_stats=True, **bufs, **kw)
        return {k: v.cpu() for k, v in r.items()}

    plain, full, zero = call(B, False), call(B, True), call(torch.zeros(N, 3), False)
    alone = model.render_frames(feat, rgba_out=torch.empty(Fn, N, 4, dtype=torch.uint8, device="cuda"), **kw)
    assert set(alone) == {"rgba_u8", "depth_map", "weights_sum"} | ({"torso_alpha_map", "torso_rgb_map", "deform"} if sc.torso else set())
    label = f"{name} {precision}"

    moved = [k for k in OTHER if k in plain and not _same(plain[k], full[k])]
    print(f"[{label}] outputs that differ when the matte is requested: {moved} (bound none)")
    assert not moved

    ws, A = full["weights_sum"], full["alpha_map"]
    ta = full["torso_alpha_map"] if sc.torso else torch.zeros_like(ws)
    assert torch.equal(A, ws + (1 - ws) * ta)
    if not sc.torso:
        assert torch.equal(A, ws)

    if gold is not None:
        for i, t in enumerate(frames):
            gws = torch.from_numpy(gold[f"f{t}_weights_sum"]).reshape(-1)
            gta = torch.from_numpy(gold[f"f{t}_torso_alpha_map"]).reshape(-1) if sc.torso else torch.zeros_like(gws)
            rep = parity_report(A[i], gws + (1 - gws) * gta, torch.from_numpy(gold[f"f{t}_knife"]))
            print(f"[{label} f{t}] coverage vs reference max|d|={rep['max_abs']:.2e} (bound {TOL_ORACLE:.0e}; all {rep['max_abs_all']:.2e}, "
                  f"knife-edge rays {rep['n_knife']})")
            assert rep["max_abs"] <= TOL_ORACLE, (label, t, rep)

    P = zero["rgb_map"]
    target = plain["rgb_map"]
    comp = P + (1 - A).unsqueeze(-1) * B
    free = (target > 0) & (target < 1)
    err = (comp - target).abs()[free].max().item()
    print(f"[{label}] |P + (1 - A) B - frame over B| max {err:.2e} (bound {TOL_COMPOSITE:.0e}) on {int(free.sum())} of {free.numel()} "
          f"unclamped channels; pixels with 0 < A < 1: {int(((A > 0) & (A < 1)).sum())}")
    assert err <= TOL_COMPOSITE, (label, err)

    rgba = full["rgba_u8"]
    assert torch.equal(rgba[..., :3], zero["rgb_u8"])
    assert torch.equal(rgba[..., 3], (A * 255).to(torch.int32).to(torch.uint8))
    assert torch.equal(alone["rgba_u8"].cpu(), rgba)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_rgba_clip_at_bench_scale(precision):
    T = 50
    sc = scn.Scene(H=512, W=512, T=T, torso=True, density_scale=8.0)
    model = build_model(sc, precision=precision)
    poses = torch.stack([sc.pose(t) for t in range(T)])
    ckw = dict(cond_feat=model.cal_cond_feat_clip(sc.cond.cuda()), bg_coords=sc.bg_coords.cuda(), T_thresh=sc.T_thresh)
    one = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, frames_per_call=T, as_rgba=True, **ckw)
    out = torch.empty(T, sc.H, sc.W, 4, dtype=torch.uint8, device="cuda")
    split = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, frames_per_call=7, as_rgba=True, out=out, **ckw)
    u8 = model.render_clip(poses, sc.intrinsics, sc.H, sc.W, frames_per_call=T, as_uint8=True, bg_color=torch.zeros(1, 3), **ckw)
    bad = [t for t in range(T) if not torch.equal(one[t], split[t])]
    cov = one[..., 3].float().mean().item() / 255
    print(f"[rgba clip T={T} 512^2 {precision}] frames of the 50-frame call equal to the frames_per_call=7 clip {T - len(bad)} of {T} "
          f"(bound {T}); mean coverage {cov:.3f}")
    assert split.data_ptr() == out.data_ptr() and split.shape == (T, sc.H * sc.W, 4)
    assert not bad, bad[:12]
    assert torch.equal(one[..., :3], u8)
    assert 0 < cov < 1


def _batch(sc, T):
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"].cuda() for f in fis], "rays_d": [f["rays_d"].cuda() for f in fis], "poses": [f["poses"].cuda() for f in fis],
            "cond_wins": [scn.cond_window(sc.cond, t, sc.hparams["smo_win_size"]).cuda() for t in range(T)],
            "bg_coords": sc.bg_coords.cuda(), "bg_img": sc.bg_color.reshape(1, -1, 3).cuda()}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("torso", [False, True], ids=["head", "torso"])
def test_driver_rgba_streamed_equals_stacked(torso, precision):
    T = 9
    sc = scn.Scene(H=64, W=64, T=T, torso=torso, density_scale=8.0)
    model = build_model(sc, precision=precision)
    batch = _batch(sc, T)
    whole = driver.render_driver_batch(model, batch, frames_per_call=4, as_rgba=True)
    chunks = [c.clone() for c in driver.iter_video_frames(model, batch, frames_per_call=4, as_rgba=True)]
    assert whole.shape == (T, 64, 64, 4) and whole.dtype == torch.uint8
    assert [tuple(c.shape) for c in chunks] == [(4, 64, 64, 4), (4, 64, 64, 4), (1, 64, 64, 4)]
    assert torch.equal(torch.cat(chunks), whole.cpu())
    # the matte does not read the batch's background
    batch["bg_img"] = torch.rand_like(batch["bg_img"])
    assert torch.equal(driver.render_driver_batch(model, batch, frames_per_call=4, as_rgba=True), whole)
