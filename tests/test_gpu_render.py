"""Fused renderer parity on the GPU (through the reference-shaped render() API and the C-ABI).

Bar (BASELINE.json north_star): rgb / alpha within 1e-3 max-abs fp32 and PSNR >= 50 dB against the CPU oracle on
identical rays and conditioning.  The tolerance is written here: TOL = 1e-3, PSNR_MIN = 50.
Discrete by-products must match exactly: the round-schedule cap B, the number of evaluated samples S and the
number of torso pixels P."""
import glob
import json
import os
import re

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from helpers import build_model, lively_state, parity_report

pytestmark = pytest.mark.gpu

TOL = 1e-3
PSNR_MIN = 50.0
GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")) if re.match(r"(head|torso)\d+_ms", os.path.basename(p)))


def _render_both(sc, state, t, oracle_ops, max_steps=None, T_thresh=None):
    from oracle.render import OracleModel
    T_thresh = sc.T_thresh if T_thresh is None else T_thresh
    hp = dict(sc.hparams)
    if max_steps is not None:
        hp["max_steps"] = max_steps
    fi = sc.frame_inputs(t)
    orc = OracleModel(state, hp)
    orc.density_scale = sc.density_scale
    ref = orc.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], T_thresh=T_thresh, **hp)
    model = build_model(sc, state)
    out = model.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda(), index=t,
                       staged=False, bg_color=fi["bg_color"].cuda(), perturb=False, force_all_rays=False, T_thresh=T_thresh, lm68=None, **hp)
    torch.cuda.synchronize()
    return ref, out, model, fi, hp


def _check(ref, out, torso, label):
    rep = parity_report(out["rgb_map"].view(-1, 3), ref["rgb_map"].view(-1, 3), ref["knife"])
    repw = parity_report(out["weights_sum"].view(-1), ref["weights_sum"].view(-1), ref["knife"])
    print(f"[{label}] rgb max|d|={rep['max_abs']:.2e} (all {rep['max_abs_all']:.2e}, knife-edge rays {rep['n_knife']}, >1e-3: {rep['n_over']}) "
          f"psnr={rep['psnr']:.1f} dB | alpha max|d|={repw['max_abs']:.2e}")
    assert rep["max_abs"] <= TOL and repw["max_abs"] <= TOL, (label, rep, repw)
    assert rep["psnr"] >= PSNR_MIN
    assert rep["n_over"] <= max(2, rep["n_knife"]), "errors above tolerance must be explained by knife-edge rays"
    d_ref, d_out = ref["depth_map"].view(-1), out["depth_map"].view(-1).cpu()
    assert torch.equal(torch.isnan(d_ref), torch.isnan(d_out))
    ok = ~torch.isnan(d_ref) & (ref["knife"].view(-1) >= 1e-3)
    assert (d_ref[ok] - d_out[ok]).abs().max().item() <= 2e-3
    if torso:
        for k in ("torso_alpha_map", "torso_rgb_map"):
            d = (out[k].cpu().reshape(-1) - ref[k].reshape(-1)).abs().max().item()
            assert d <= TOL, (label, k, d)
        if "deform" in ref:
            assert out["deform"].shape == ref["deform"].shape
            assert (out["deform"].cpu() - ref["deform"]).abs().max().item() <= 1e-4


CASES = [
    # name, torso, size, max_steps, density_scale, lively gain (None = SURVEY 8(d) default-init scene), table decay
    ("head_default_ds1", False, 64, 16, 1.0, None, 0.0),
    ("head_default_ms8", False, 64, 8, 1.0, None, 0.0),
    ("head_lively_ds1", False, 64, 16, 1.0, 4.0, 1.0),
    ("head_lively_ds16", False, 64, 16, 16.0, 4.0, 1.0),
    ("head_lively_ds64_ragged", False, 50, 16, 64.0, 4.0, 1.0),
    ("torso_default_ds1", True, 64, 16, 1.0, None, 0.0),
    ("torso_lively_ds8", True, 64, 16, 8.0, 3.0, 1.0),
    ("torso_lively_ms1024", True, 40, 1024, 8.0, 3.0, 1.0),
]


@pytest.mark.parametrize("name,torso,size,max_steps,ds,gain,decay", CASES, ids=[c[0] for c in CASES])
def test_render_matches_oracle(oracle_ops, name, torso, size, max_steps, ds, gain, decay):
    sc = scn.Scene(H=size, W=size, T=8, torso=torso, max_steps=max_steps, density_scale=ds, table_decay=decay,
                   table_amp=1.0 if decay else 0.5)
    state = lively_state(sc.state, gain) if gain else sc.state
    for t in (0, 5):
        ref, out, model, fi, hp = _render_both(sc, state, t, oracle_ops)
        _check(ref, out, torso, f"{name}/f{t}")
        # discrete by-products: exact
        res = model.render_frames(model.cal_cond_feat(fi["cond"].cuda()).view(1, -1), rays_o=fi["rays_o"].cuda(), rays_d=fi["rays_d"].cuda(),
                                  pose6=fi["poses"].cuda() if torso else None, bg_coords=fi["bg_coords"].cuda() if torso else None,
                                  bg_color=fi["bg_color"].cuda(), dt_gamma=hp["dt_gamma"], max_steps=hp["max_steps"], T_thresh=sc.T_thresh, want_stats=True)
        st = res["stats"][0].tolist()
        n_knife = int((ref["knife"] < 1e-3).sum())
        if ref["stats"]["schedule"][-1][0] > 0 and sum(s for _, s in ref["stats"]["schedule"]) >= hp["max_steps"]:
            assert st[0] == ref["stats"]["B_total"], (st, ref["stats"])
        assert abs(st[2] - ref["stats"]["S"]) <= n_knife + 2 * 0, (st, ref["stats"]["S"], n_knife)
        assert st[3] == ref["stats"]["P"]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_render_matches_reference_golden(path):
    """Against the committed outputs of the REFERENCE's own render() (CPU, fp32)."""
    z = np.load(path)
    m = json.loads(bytes(z["meta"]).decode())
    sc = scn.Scene(H=m["size"], W=m["size"], T=8, torso=m["torso"], max_steps=m["max_steps"], density_scale=m["density_scale"])
    model = build_model(sc)
    for t in m["frames"]:
        fi = sc.frame_inputs(t)
        out = model.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda(),
                           bg_color=fi["bg_color"].cuda(), T_thresh=m["T_thresh"], **sc.hparams)
        knife = torch.from_numpy(z[f"f{t}_knife"])
        rep = parity_report(out["rgb_map"].view(-1, 3), torch.from_numpy(z[f"f{t}_rgb_map"]).view(-1, 3), knife)
        print(f"[golden {m['name']}/f{t}] max|d|={rep['max_abs']:.2e} psnr={rep['psnr']:.1f}")
        assert rep["max_abs"] <= TOL and rep["psnr"] >= PSNR_MIN


def test_bg_color_none_and_head_only_epilogue(oracle_ops):
    from oracle.render import OracleModel
    sc = scn.Scene(H=48, W=48, T=4, torso=False, density_scale=8.0)
    fi = sc.frame_inputs(2)
    orc = OracleModel(sc.state, sc.hparams); orc.density_scale = 8.0
    ref = orc.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=None, T_thresh=0.01, **sc.hparams)
    model = build_model(sc)
    out = model.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda(), bg_color=None, T_thresh=0.01, **sc.hparams)
    assert (out["rgb_map"].cpu() - ref["rgb_map"]).abs().max().item() <= TOL
    assert out["rgb_map"].shape == ref["rgb_map"].shape and out["depth_map"].shape == ref["depth_map"].shape


def test_rays_missing_the_volume(oracle_ops):
    """Edge case: camera looking away => every ray misses the aabb: image == background, depth NaN like the reference."""
    from oracle.render import OracleModel
    sc = scn.Scene(H=32, W=32, T=2, torso=False)
    fi = sc.frame_inputs(0)
    ro = fi["rays_o"].clone(); ro[..., 1] += 6.0
    orc = OracleModel(sc.state, sc.hparams)
    ref = orc.render(ro, fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], T_thresh=0.01, **sc.hparams)
    model = build_model(sc)
    out = model.render(ro.cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda(), bg_color=fi["bg_color"].cuda(), T_thresh=0.01, **sc.hparams)
    assert torch.equal(out["rgb_map"].cpu(), ref["rgb_map"])
    assert torch.isnan(ref["depth_map"]).all() and torch.isnan(out["depth_map"]).all()
    assert (out["weights_sum"] == 0).all()


def test_clip_api_equals_per_frame_render_and_is_deterministic():
    sc = scn.Scene(H=64, W=64, T=6, torso=True, density_scale=8.0, table_decay=1.0, table_amp=1.0)
    model = build_model(sc, lively_state(sc.state, 3.0))
    poses = torch.stack([sc.pose(t) for t in range(sc.T)])
    rgb = model.render_clip(poses, sc.intrinsics, 64, 64, cond_seq=sc.cond, bg_color=sc.bg_color, bg_coords=sc.bg_coords, T_thresh=0.01, frames_per_call=4)
    rgb2 = model.render_clip(poses, sc.intrinsics, 64, 64, cond_seq=sc.cond, bg_color=sc.bg_color, bg_coords=sc.bg_coords, T_thresh=0.01, frames_per_call=6)
    assert torch.equal(rgb, rgb2), "frames must not depend on how the clip is batched (or on slot scheduling)"
    for t in (0, 3, 5):
        fi = sc.frame_inputs(t)
        out = model.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda(),
                           bg_color=fi["bg_color"].cuda(), T_thresh=0.01, **sc.hparams)
        # in-kernel ray generation vs torch get_rays: 1-ulp ray differences may flip a cell at a few pixels
        d = (rgb[t] - out["rgb_map"].view(-1, 3)).abs().max(-1).values
        print(f"[clip vs per-frame f{t}] max {d.max().item():.2e}, frac>1e-3 {(d > 1e-3).float().mean().item():.2e}")
        assert (d > 1e-3).float().mean().item() < 2e-3, (t, d.max().item())
        assert d.median().item() < 1e-5


def test_full_size_properties():
    """512x512 (BASELINE size): size-independent properties instead of a full CPU oracle run."""
    sc = scn.Scene(H=512, W=512, T=2, torso=True, density_scale=8.0)
    model = build_model(sc)
    fi = sc.frame_inputs(0)
    args = (fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda())
    a = model.render(*args, bg_color=fi["bg_color"].cuda(), T_thresh=0.01, **sc.hparams)
    b = model.render(*args, bg_color=fi["bg_color"].cuda(), T_thresh=0.01, **sc.hparams)
    assert torch.equal(a["rgb_map"], b["rgb_map"]) and torch.equal(a["weights_sum"], b["weights_sum"])   # deterministic
    rgb, ws = a["rgb_map"].view(-1, 3), a["weights_sum"].view(-1)
    assert rgb.min().item() >= 0 and rgb.max().item() <= 1 and ws.min().item() >= 0 and ws.max().item() <= 1 + 1e-5
    # linearity in the background: image(bg) - image(0) == (1 - ws) * bg' where bg' only changes outside the torso
    z = model.render(*args, bg_color=torch.zeros_like(fi["bg_color"]).cuda(), T_thresh=0.01, **sc.hparams)
    ta = a["torso_alpha_map"].view(-1, 1)
    expect = (1 - ws).unsqueeze(-1) * (fi["bg_color"].cuda().view(-1, 3) * (1 - ta))
    assert ((rgb - z["rgb_map"].view(-1, 3)) - expect).abs().max().item() < 1e-5
    # the 64x64 render is a subsampling-consistent view: centre pixel rays of the ellipsoid are opaque-ish, corners are background
    assert ws.view(512, 512)[256, 256].item() > 0.5 and ws.view(512, 512)[2, 2].item() == 0
