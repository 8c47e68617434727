"""The torso occupancy-grid refresh on the GPU (k_torso_query / k_torso_sr_query in torso_grid_kernel.cu, k_torso_dilate_ema in
grid_kernels.cu, gfpp.h section F) against the reference's own update_extra_state (tests/golden/torso_*grid*.npz) and the CPU oracle.

The torso fields run in fp32 FFMA and their alphas are sigmoids in [0,1]; the device sums the mean in double in a fixed order, the
reference in fp32.  The bounds are about twice the errors the first H100 run measured (raw 8.3e-7, EMA 6.0e-7, mean 7.1e-8 relative;
forward_torso 7.7e-7 on the colour against the fp32 oracle).  Every error is printed."""
import ctypes
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams, may_intrinsics
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR
from oracle import make_torso_grid_golden as mtg
from oracle.render import OracleModel

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _model(kind, H):
    inp = mtg.inputs(kind, H)
    m = (RADNeRFTorsowithSR if kind == "torso_sr" else RADNeRFTorso)(inp["hp"])
    m.load_state_dict(inp["state"], strict=True)
    m.poses, m.lm68s = inp["poses"], inp["lm68s"]
    return m.cuda().eval(), inp


def _cond(kind, g):
    return torch.from_numpy(g["lm68"] if kind == "torso_sr" else g["pose6"])


@pytest.mark.parametrize("name", list(mtg.CASES))
def test_refresh_vs_reference(name):
    kind, H = mtg.CASES[name]
    g = np.load(os.path.join(GOLDEN, name))
    m, inp = _model(kind, H)
    tmp = torch.empty(H * H, device="cuda")
    mean = m.refresh_torso_grid(_cond(kind, g), inp["code"], inp["noise"], mtg.DECAY, tmp_grid=tmp)
    torch.cuda.synchronize()
    d_raw = (tmp.cpu() - torch.from_numpy(g["raw"])).abs().max().item()
    d_ema = (m.density_grid_torso.cpu() - torch.from_numpy(g["ema"])).abs().max().item()
    gm = float(g["mean"][0])
    d_mean = abs(mean.item() - gm) / gm
    print(f"[torso refresh {name}] max|gpu - reference| raw {d_raw:.3e}, EMA {d_ema:.3e}; rel mean {d_mean:.3e}; "
          f"{m.last_launch_count} launches")
    assert d_raw <= 2e-6 and d_ema <= 2e-6 and d_mean <= 2e-7


def test_forward_torso_vs_oracle(oracle_ops):
    inp = mtg.inputs("torso", 128)
    m, _ = _model("torso", 128)
    x = scn.hashed_uniform(2 * 65536, 23, 2.0).view(-1, 2)
    pose6 = scn.convert_poses(scn.camera_pose(3).view(1, 4, 4))
    code = inp["state"]["torso_individual_codes"][2:3]
    a, c, dx = m.forward_torso(x.cuda(), pose6.cuda(), code.cuda())
    torch.cuda.synchronize()
    orc = OracleModel(inp["state"], inp["hp"], torso=True)
    ra, rc, rdx = orc.forward_torso(x, pose6, code)
    da, dc, dd = [(u.cpu() - v).abs().max().item() for u, v in ((a, ra), (c, rc), (dx, rdx))]
    print(f"[forward_torso] 65536 points: max|gpu - oracle| alpha {da:.3e}, color {dc:.3e}, dx {dd:.3e}")
    assert a.shape == (65536, 1) and c.shape == (65536, 3) and dx.shape == (65536, 2)
    assert da <= 2e-6 and dc <= 2e-6 and dd <= 2e-6


@pytest.mark.parametrize("name", list(mtg.CASES))
def test_update_extra_state_vs_reference(name):
    """The whole update_extra_state, conditioning included (the training pose converted by scene.convert_poses / the lm68s row and
    the torso code row `pose_index` picks), against the reference's own call on the same pose index."""
    kind, H = mtg.CASES[name]
    g = np.load(os.path.join(GOLDEN, name))
    m, inp = _model(kind, H)
    m.update_extra_state(decay=mtg.DECAY, pose_index=int(g["pose_index"][0]), noise=inp["noise"])
    d_ema = (m.density_grid_torso.cpu() - torch.from_numpy(g["ema"])).abs().max().item()
    gm = float(g["mean"][0])
    d_mean = abs(m.mean_density_torso - gm) / gm
    print(f"[update_extra_state {name}] max|gpu - reference| EMA {d_ema:.3e}; rel mean {d_mean:.3e}")
    assert d_ema <= 2e-6 and d_mean <= 2e-7


@pytest.mark.parametrize("kind", ["torso", "torso_sr"])
def test_refresh_is_deterministic(kind):
    name = {"torso": "torso_grid128.npz", "torso_sr": "torso_sr_grid128.npz"}[kind]
    g = np.load(os.path.join(GOLDEN, name))
    outs = []
    for _ in range(2):
        m, inp = _model(kind, 128)
        tmp = torch.empty(128 * 128, device="cuda")
        mean = m.refresh_torso_grid(_cond(kind, g), inp["code"], inp["noise"], mtg.DECAY, tmp_grid=tmp)
        outs.append((m.density_grid_torso.clone(), mean.clone(), tmp))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))


def test_short_workspace_is_refused():
    m, inp = _model("torso", 32)
    _, _, model, _ = m._ensure_packed()
    L = _capi.lib()
    need = L.gfpp_torso_grid_workspace_bytes(32)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    pose6, code = torch.zeros(6, device="cuda"), inp["code"].cuda()
    noise, mean, xy, out = inp["noise"].cuda(), torch.empty(1, device="cuda"), torch.zeros(8, 2, device="cuda"), torch.empty(8, device="cuda")
    rc = L.gfpp_torso_grid_update(ctypes.byref(model), pose6.data_ptr(), code.data_ptr(), noise.data_ptr(), 0.95, m.density_grid_torso.data_ptr(),
                                  mean.data_ptr(), None, ws.data_ptr(), need - 1, _capi.stream_ptr())
    assert rc == -3 and b"workspace" in L.gfpp_last_error()
    rc = L.gfpp_torso_query(ctypes.byref(model), xy.data_ptr(), 8, pose6.data_ptr(), code.data_ptr(), out.data_ptr(), None, None,
                            ws.data_ptr(), L.gfpp_torso_query_workspace_bytes() - 1, _capi.stream_ptr())
    assert rc == -3 and b"workspace" in L.gfpp_last_error()
    sr, sinp = _model("torso_sr", 32)
    st = sr._torso_native_state()
    lm68 = sinp["lm68s"][0].cuda()
    rc = L.gfpp_torso_sr_grid_update(ctypes.byref(st["model"]), lm68.data_ptr(), code.data_ptr(), noise.data_ptr(), 0.95,
                                     sr.density_grid_torso.data_ptr(), mean.data_ptr(), None, ws.data_ptr(), need - 1, _capi.stream_ptr())
    assert rc == -3 and b"workspace" in L.gfpp_last_error()


def _fresh(cls, hp, m, mean):
    f = cls(hp)
    f.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    f.mean_density_torso = mean
    return f


def test_torso_render_after_update_matches_a_fresh_model():
    """update_extra_state writes density_grid_torso in place and the new threshold into the packed handle; the next render_clip
    must be the one a model packed from the updated state renders, bit for bit, and must differ from the one before."""
    sc = scn.Scene(H=64, W=64, T=2, torso=True, density_scale=8.0)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale, m.poses = sc.density_scale, torch.stack([sc.pose(t) for t in range(4)])
    m = m.cuda().eval()
    poses = torch.stack([sc.pose(t) for t in range(2)]).cuda()
    kw = dict(cond_seq=sc.cond.cuda(), bg_color=sc.bg_color.cuda(), bg_coords=sc.bg_coords.cuda(), T_thresh=sc.T_thresh)
    before = m.render_clip(poses, sc.intrinsics, 64, 64, **kw)
    packed_before = m._packed[1]
    noise = (scn.hashed_uniform(128 * 128 * 2, 7, 1.0) + 0.5).view(128, 128, 2)
    m.update_extra_state(pose_index=2, noise=noise)
    after = m.render_clip(poses, sc.intrinsics, 64, 64, **kw)
    assert m._packed[1] is packed_before                      # not repacked
    fresh = _fresh(RADNeRFTorso, sc.hparams, m, m.mean_density_torso)
    fresh.density_scale = sc.density_scale
    ref = fresh.cuda().eval().render_clip(poses, sc.intrinsics, 64, 64, **kw)
    torch.cuda.synchronize()
    print(f"[torso render after update] mean_density_torso {m.mean_density_torso:.4f}; pixels changed by the refresh "
          f"{int((after != before).any(-1).sum())}; max|after - fresh model| {(after - ref).abs().max().item():.3e}")
    assert torch.equal(after, ref) and bool((after != before).any())


def test_torso_sr_render_after_update_matches_a_fresh_model():
    hp = may_hparams(**mtg.SR_OVERRIDES)
    state = scn.make_torso_sr_state(hp)
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(state, strict=True)
    m.density_scale, m.poses, m.lm68s = 8.0, torch.stack([scn.camera_pose(t) for t in range(4)]), scn.lm68_sequence(4)
    m = m.cuda().eval()
    poses = m.poses[:1].cuda()
    intr = may_intrinsics(256, 256)
    kw = dict(cond_seq=scn.cond_sequence(1).cuda(), bg_coords=scn.get_bg_coords(256, 256).cuda(), lm68_seq=m.lm68s[:1].cuda(),
              sr_noise_mode="const", T_thresh=0.01)
    before = m.render_clip(poses, intr, 256, 256, **kw)
    st_before, packed_before = m._torso_native_state(), m._packed[1]
    noise = (scn.hashed_uniform(128 * 128 * 2, 7, 1.0) + 0.5).view(128, 128, 2)
    m.update_extra_state(pose_index=2, noise=noise)
    after = m.render_clip(poses, intr, 256, 256, **kw)
    assert m._torso_native_state() is st_before and m._packed[1] is packed_before      # neither handle repacked
    fresh = _fresh(RADNeRFTorsowithSR, hp, m, m.mean_density_torso)
    fresh.density_scale = 8.0
    ref = fresh.cuda().eval().render_clip(poses, intr, 256, 256, **kw)
    torch.cuda.synchronize()
    print(f"[torso-SR render after update] mean_density_torso {m.mean_density_torso:.4f}; max|after - before| "
          f"{(after - before).abs().max().item():.3e}; max|after - fresh model| {(after - ref).abs().max().item():.3e}")
    assert torch.equal(after, ref) and bool((after != before).any())
