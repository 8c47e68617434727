"""Video frames from the SR checkpoints on the GPU: the uint8 epilogue of the SR head's last kernel (gfpp_sr_forward_video), the
SR models' render_clip(as_uint8=True), render_driver_batch and iter_video_frames for all four model classes.

Every uint8 frame must be BIT-IDENTICAL to `to_uint8` of the fp32 frame the same computation gives: the epilogue applies the
driver's `(rgb * 255).int()` to the very clamped fp32 value it would store, and the fp32 frame of the new entry point is the
one gfpp_sr_forward writes."""
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import driver
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.dist import to_uint8
from genefaceplusplus_b200.superres import Superresolution
from helpers import build_model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
R = 256


@pytest.fixture(scope="module")
def sr_net():
    g = np.load(os.path.join(GOLD, "sr_head.npz"))
    meta = json.loads(bytes(g["meta"]).decode())
    net = Superresolution(channels=3).eval()
    net.load_state_dict(scn.synthetic_sr_state({k: tuple(v) for k, v in meta["shapes"].items()}, seed=3), strict=False)
    return net.cuda()


def _frames(F):
    base = scn.hashed_uniform(R * R * 3, 78, 1.0).reshape(R, R, 3) + 0.5
    fr = [base.flip(f % 2).roll(17 * f, 1) * (1.0 - 0.05 * f) for f in range(F)]
    return torch.stack(fr).reshape(F, R * R, 3).contiguous().cuda()


@pytest.mark.parametrize("mode", ["none", "const", "planes"])
@pytest.mark.parametrize("F", [1, 3, 8, 9])
def test_sr_uint8_epilogue_is_bit_identical(sr_net, F, mode):
    x = _frames(F)
    kw = {"noise_mode": "none" if mode == "none" else "const", "frames_per_call": 16, "clamp": True}
    if mode == "planes":          # one plane per frame and layer, as noise_mode='random' hands them over
        gen = torch.Generator().manual_seed(F)
        kw["noise_planes"] = [(torch.randn(F, l.resolution, l.resolution, generator=gen) * 0.05).cuda() for l in sr_net._layers()]
    ref = sr_net.forward_native(x, **kw)                                        # gfpp_sr_forward, clamp01 = 1
    both32 = torch.full_like(ref, float("nan"))
    both8 = torch.full((F, 2 * R, 2 * R, 3), 0xAB, dtype=torch.uint8, device="cuda")
    got = sr_net.forward_native(x, out=both32, u8_out=both8, **kw)              # gfpp_sr_forward_video, both outputs
    only8 = torch.full_like(both8, 0x5C)
    got8 = sr_net.forward_native(x, u8_out=only8, **kw)                         # uint8 only: no fp32 frame
    torch.cuda.synchronize()
    assert got is both8 and got8 is only8
    assert torch.equal(both32, ref), "fp32 output of gfpp_sr_forward_video differs from gfpp_sr_forward"
    want = to_uint8(ref.permute(0, 2, 3, 1))
    assert torch.equal(both8, want) and torch.equal(only8, want)
    print(f"F={F} {mode}: {int((want == 0).sum())} zero and {int((want == 255).sum())} saturated channel values of {want.numel()}")


def test_sr_uint8_rejects_unclamped_or_misshaped_buffers(sr_net):
    x = _frames(2)
    with pytest.raises(ValueError):
        sr_net.forward_native(x, clamp=False, u8_out=torch.empty(2, 2 * R, 2 * R, 3, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        sr_net.forward_native(x, clamp=True, u8_out=torch.empty(2, 3, 2 * R, 2 * R, dtype=torch.uint8, device="cuda"))


# ------------------------------------------------------------------------------------------------ SR model classes
def _head_sr():
    from genefaceplusplus_b200.renderer import RADNeRFwithSR
    meta = json.loads(bytes(np.load(os.path.join(GOLD, "head_sr256.npz"))["meta"]).decode())
    hp = may_hparams(**{**meta["overrides"], "max_steps": 16})
    m = RADNeRFwithSR(hp)
    m.load_state_dict(scn.make_head_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    return m.cuda().eval(), meta


def _torso_sr():
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
    meta = json.loads(bytes(np.load(os.path.join(GOLD, "torso_sr256.npz"))["meta"]).decode())
    hp = may_hparams(**{**meta["overrides"], "torso_head_aware": True, "max_steps": 16})
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    return m.cuda().eval(), meta


def _model(which):
    if which == "head_sr":
        return _head_sr()
    if which == "torso_sr":
        return _torso_sr()
    sc = scn.Scene(H=64, W=64, T=2, torso=which == "torso", max_steps=16)
    return build_model(sc), None


def _batch(m, which, T):
    """The driver's batch (genefacepp_infer.py:203-269, 400-429) on the GPU: per-frame rays, windows, poses, eye values, lm68."""
    H = R if which in ("head_sr", "torso_sr") else 64
    sc = scn.Scene(H=H, W=H, T=T, torso=which in ("torso", "torso_sr"), max_steps=16)
    fis = [sc.frame_inputs(t) for t in range(T)]
    eye = 0.3
    return sc, {"rays_o": [f["rays_o"].cuda() for f in fis], "rays_d": [f["rays_d"].cuda() for f in fis],
                "poses": [f["poses"].cuda() for f in fis], "cond_wins": [scn.cond_window(sc.cond, t, m.smo_win_size).cuda() for t in range(T)],
                "bg_coords": sc.bg_coords.cuda(), "bg_img": sc.bg_color.reshape(1, -1, 3).cuda(),
                "eye_area_percent": (eye + 0.05 * torch.arange(T, dtype=torch.float32)).reshape(T, 1).cuda(),
                "lm68": scn.lm68_sequence(T).cuda()}


@pytest.mark.parametrize("mode", ["const", "none"])
@pytest.mark.parametrize("which", ["head_sr", "torso_sr"])
def test_sr_render_clip_as_uint8(which, mode):
    m, meta = _model(which)
    T = 5
    sc = scn.Scene(H=R, W=R, T=T, torso=which == "torso_sr")
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    kw = {"cond_seq": sc.cond.cuda(), "eye_area_percent": torch.full((T,), meta["eye"]), "max_steps": 16, "T_thresh": sc.T_thresh,
          "sr_noise_mode": mode}
    if which == "torso_sr":
        kw.update(bg_color=sc.bg_color.cuda(), bg_coords=sc.bg_coords.cuda(), lm68_seq=scn.lm68_sequence(T).cuda(), frames_per_call=2)
    else:
        kw.update(bg_color=sc.bg_color.cuda().reshape(-1, 3), sr_frames_per_call=2)
    f32 = m.render_clip(poses, sc.intrinsics, R, R, **kw)
    u8 = m.render_clip(poses, sc.intrinsics, R, R, as_uint8=True, **kw)
    buf = torch.full((T, 2 * R, 2 * R, 3), 0x33, dtype=torch.uint8, device="cuda")
    into = m.render_clip(poses, sc.intrinsics, R, R, as_uint8=True, out=buf, **kw)
    torch.cuda.synchronize()
    assert f32.shape == (T, 3, 2 * R, 2 * R) and u8.shape == (T, 2 * R, 2 * R, 3) and u8.dtype == torch.uint8
    assert into.data_ptr() == buf.data_ptr()
    want = to_uint8(f32.permute(0, 2, 3, 1))
    assert torch.equal(u8, want) and torch.equal(buf, want)


def _per_frame(m, batch, t, feat, noise_mode):
    """The driver's frame t (genefacepp_infer.py:476-481): render(...)["sr_rgb_map"][0].  cal_cond_feat is pinned to the batched
    conditioning row the shim computes (render_driver_batch runs the conditioning nets over the whole clip at once, which equals
    the per-frame nets to 1e-6 -- checked below -- but not to the bit)."""
    m.cal_cond_feat = lambda cond, eye_area_percent=None: feat[t]
    try:
        hp = {k: v for k, v in m.hparams.items() if k not in ("max_steps", "dt_gamma", "bg_color")}
        res = m.render(batch["rays_o"][t], batch["rays_d"][t], batch["cond_wins"][t], batch["bg_coords"], batch["poses"][t], index=t,
                       staged=False, bg_color=batch["bg_img"], lm68=batch["lm68"][t], perturb=False, force_all_rays=False, T_thresh=0.01,
                       eye_area_percent=batch["eye_area_percent"][t], dt_gamma=m.hparams["dt_gamma"], max_steps=16, sr_noise_mode=noise_mode,
                       **hp)
    finally:
        del m.cal_cond_feat
    return res["sr_rgb_map"][0]


@pytest.mark.parametrize("which", ["head_sr", "torso_sr"])
def test_driver_batch_sr_equals_per_frame_render(which):
    m, _ = _model(which)
    T = 9
    _, batch = _batch(m, which, T)
    feat = driver.cond_feat_from_windows(m, batch["cond_wins"], batch["eye_area_percent"])
    for t in range(T):
        one = m.cal_cond_feat(batch["cond_wins"][t], eye_area_percent=batch["eye_area_percent"][t])
        assert (feat[t] - one.reshape(-1)).abs().max().item() < 1e-6
    got = driver.render_driver_batch(m, batch, T_thresh=0.01, frames_per_call=4, sr_noise_mode="const")
    u8 = driver.render_driver_batch(m, batch, T_thresh=0.01, frames_per_call=4, sr_noise_mode="const", as_uint8=True)
    ref = torch.stack([_per_frame(m, batch, t, feat, "const") for t in range(T)])
    torch.cuda.synchronize()
    assert got.shape == (T, 3, 2 * R, 2 * R) and got.dtype == torch.float32
    for t in range(T):
        assert torch.equal(got[t], ref[t]), f"frame {t}: max |driver - render()| = {(got[t] - ref[t]).abs().max().item():.3e}"
    assert torch.equal(u8, to_uint8(got.permute(0, 2, 3, 1)))
    # 'random' (the driver's own default): one noise plane per frame and layer, drawn by the SR head
    with torch.no_grad():
        for lay in m.sr_net._layers():
            lay.noise_strength.fill_(0.05)
    const = driver.render_driver_batch(m, batch, T_thresh=0.01, frames_per_call=4, sr_noise_mode="const")
    rnd = driver.render_driver_batch(m, batch, T_thresh=0.01, frames_per_call=4, sr_noise_mode="random")
    rnd8 = driver.render_driver_batch(m, batch, T_thresh=0.01, frames_per_call=4, sr_noise_mode="random", as_uint8=True)
    torch.cuda.synchronize()
    assert rnd.shape == const.shape and rnd8.shape == (T, 2 * R, 2 * R, 3)
    assert 0.0 <= rnd.min().item() and rnd.max().item() <= 1.0
    for t in range(T):
        assert not torch.equal(rnd[t], const[t]) and not torch.equal(rnd8[t], to_uint8(const[t].permute(1, 2, 0)))


@pytest.mark.parametrize("which", ["head", "torso", "head_sr", "torso_sr"])
def test_iter_video_frames_equals_the_uint8_clip(which):
    m, _ = _model(which)
    T = 11
    _, batch = _batch(m, which, T)
    kw = {"T_thresh": 0.01, "sr_noise_mode": "const"}
    whole = driver.render_driver_batch(m, batch, frames_per_call=4, as_uint8=True, **kw)
    if which in ("head", "torso"):     # the non-SR epilogue's uint8 frames are to_uint8 of its fp32 frames
        assert torch.equal(whole, driver.video_uint8(driver.render_driver_batch(m, batch, frames_per_call=4, **kw)))
    chunks = []
    for c in driver.iter_video_frames(m, batch, frames_per_call=4, **kw):
        assert c.device.type == "cpu" and c.is_pinned() and c.dtype == torch.uint8
        chunks.append(c.clone())
    assert [c.shape[0] for c in chunks] == [4, 4, 3]
    assert torch.equal(torch.cat(chunks), whole.cpu())

    # closed after its first chunk: the queued work is finished by close(), and the next render is unaffected
    gen = driver.iter_video_frames(m, batch, frames_per_call=4, **kw)
    first = next(gen).clone()
    gen.close()
    torch.cuda.synchronize()
    assert torch.equal(first, whole[:4].cpu())
    again = torch.cat([c.clone() for c in driver.iter_video_frames(m, batch, frames_per_call=4, **kw)])
    assert torch.equal(again, whole.cpu())
    assert torch.equal(driver.render_driver_batch(m, batch, frames_per_call=4, as_uint8=True, **kw), whole)
