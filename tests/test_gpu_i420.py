"""Planar I420 video frames on the GPU: gfpp_rgb_u8_to_i420 (include/gfpp.h section N) and the as_yuv420 clip and driver APIs of
all four model classes.

Every I420 byte must be BIT-IDENTICAL to video.i420_reference, the numpy restatement of the header's integer formulas, applied to
the uint8 frames the same seeded call gives with as_uint8=True: the conversion reads those very frames, and the I420 path draws
the SR head's noise planes exactly as the uint8 path does."""
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import driver, video
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from helpers import build_model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
PRECISIONS = ["fp32", "fp16", "robust", "bf16x3", "bf16"]
R = 256


def _ref(u8, H, W):
    """video.i420_reference of uint8 frames [F,H,W,3] or [F,H*W,3] on any device -> CPU uint8 [F,H*W*3/2]."""
    return torch.from_numpy(video.i420_reference(u8.cpu().reshape(-1, H, W, 3).numpy()))


# ------------------------------------------------------------------------------------------------ the kernel
def _random_frames(F, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, generator=g)
    x[0, 0] = 0                                                  # both ends of the range in every frame set
    x[-1, -1] = 255
    if H >= 4 and W >= 4:
        x[:, :2, :2] = 255                                       # a saturated block and a black one
        x[:, -2:, -2:] = 0
    return x


@pytest.mark.parametrize("F", [1, 3])
@pytest.mark.parametrize("H", [2, 4, 512])
@pytest.mark.parametrize("W", [2, 6, 510, 512])
def test_kernel_is_bit_identical_to_the_restatement(F, H, W):
    rgb = _random_frames(F, H, W, seed=F * 10007 + H * 31 + W)
    want = _ref(rgb, H, W)
    fb = H * W * 3 // 2
    dev = rgb.cuda()
    got = video.rgb_u8_to_i420(dev, H, W)
    assert got.shape == (F, fb) and got.dtype == torch.uint8
    assert torch.equal(got.cpu(), want)
    # `out` and the input at aligned and unaligned offsets inside larger buffers: the 32-bit kernel where both are 4-byte aligned and
    # W % 4 == 0, the byte kernel otherwise; the bytes around `out` stay untouched
    n_in = F * H * W * 3
    for off_in, off_out in ((0, 1), (1, 0), (2, 3), (4, 4)):
        src = torch.full((n_in + 8,), 0x5A, dtype=torch.uint8, device="cuda")
        src[off_in:off_in + n_in] = dev.reshape(-1)
        big = torch.full((F * fb + 8,), 0xA5, dtype=torch.uint8, device="cuda")
        out = big[off_out:off_out + F * fb].view(F, fb)
        r = video.rgb_u8_to_i420(src[off_in:off_in + n_in], H, W, out=out)
        assert r.data_ptr() == out.data_ptr()
        host = big.cpu()
        assert torch.equal(host[off_out:off_out + F * fb].view(F, fb), want), (off_in, off_out)
        assert (host[:off_out] == 0xA5).all() and (host[off_out + F * fb:] == 0xA5).all(), (off_in, off_out)


def test_kernel_many_frames_on_the_current_stream():
    F, H, W = 37, 96, 128
    rgb = _random_frames(F, H, W, seed=5)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dev = rgb.cuda(non_blocking=False)
        got = video.rgb_u8_to_i420(dev, H, W)
    s.synchronize()
    assert torch.equal(got.cpu(), _ref(rgb, H, W))


# ------------------------------------------------------------------------------------------------ render_clip: head and torso
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("torso", [False, True], ids=["head", "torso"])
def test_render_clip_as_yuv420_equals_the_uint8_clip(torso, precision):
    H, W, T = 48, 64, 7                                          # not square: a swapped H and W shows
    sc = scn.Scene(H=H, W=W, T=T, torso=torso, density_scale=8.0)
    model = build_model(sc, precision=precision)
    poses = torch.stack([sc.pose(t) for t in range(T)])
    kw = dict(cond_feat=model.cal_cond_feat_clip(sc.cond.cuda()), bg_coords=sc.bg_coords.cuda() if torso else None, T_thresh=sc.T_thresh,
              bg_color=sc.bg_color.cuda())
    u8 = model.render_clip(poses, sc.intrinsics, H, W, frames_per_call=3, as_uint8=True, **kw)
    want = _ref(u8, H, W)
    buf = torch.full((T, H * W * 3 // 2), 0x33, dtype=torch.uint8, device="cuda")
    got = model.render_clip(poses, sc.intrinsics, H, W, frames_per_call=3, as_yuv420=True, out=buf, **kw)   # 3 + 3 + 1 frames
    assert got.data_ptr() == buf.data_ptr() and got.shape == (T, H * W * 3 // 2) and got.dtype == torch.uint8
    assert torch.equal(got.cpu(), want)
    one = model.render_clip(poses, sc.intrinsics, H, W, frames_per_call=T, as_yuv420=True, **kw)
    assert torch.equal(one.cpu(), want)
    # `out` reused by a second call with another background
    kw["bg_color"] = torch.rand(H * W, 3, generator=torch.Generator().manual_seed(2)).cuda()
    u8b = model.render_clip(poses, sc.intrinsics, H, W, frames_per_call=3, as_uint8=True, **kw)
    again = model.render_clip(poses, sc.intrinsics, H, W, frames_per_call=3, as_yuv420=True, out=buf, **kw)
    assert again.data_ptr() == buf.data_ptr() and not torch.equal(u8b, u8)
    assert torch.equal(buf.cpu(), _ref(u8b, H, W))


# ------------------------------------------------------------------------------------------------ SR classes
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


def _noisy(m):
    """Non-zero noise strengths, so that 'random' draws planes that change the frames (the synthetic states have zero strengths)."""
    with torch.no_grad():
        for lay in m.sr_net._layers():
            lay.noise_strength.fill_(0.05)
    return m


@pytest.mark.parametrize("mode", ["random", "const"])
@pytest.mark.parametrize("which", ["head_sr", "torso_sr"])
def test_sr_render_clip_as_yuv420_equals_the_uint8_clip(which, mode):
    m, meta = _head_sr() if which == "head_sr" else _torso_sr()
    _noisy(m)
    T, S = 5, 2 * R
    sc = scn.Scene(H=R, W=R, T=T, torso=which == "torso_sr")
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    kw = {"cond_seq": sc.cond.cuda(), "eye_area_percent": torch.full((T,), meta["eye"]), "max_steps": 16, "T_thresh": sc.T_thresh,
          "sr_noise_mode": mode}
    if which == "torso_sr":
        kw.update(bg_color=sc.bg_color.cuda(), bg_coords=sc.bg_coords.cuda(), lm68_seq=scn.lm68_sequence(T).cuda(), frames_per_call=2)
    else:
        kw.update(bg_color=sc.bg_color.cuda().reshape(-1, 3), sr_frames_per_call=2)

    def clip(seed, **extra):
        torch.manual_seed(seed)
        return m.render_clip(poses, sc.intrinsics, R, R, **kw, **extra)

    u8 = clip(7, as_uint8=True)
    want = _ref(u8, S, S)
    buf = torch.full((T, S * S * 3 // 2), 0x33, dtype=torch.uint8, device="cuda")
    got = clip(7, as_yuv420=True, out=buf)
    torch.cuda.synchronize()
    assert got.data_ptr() == buf.data_ptr() and got.shape == (T, S * S * 3 // 2)
    assert torch.equal(got.cpu(), want)
    assert torch.equal(clip(7, as_yuv420=True).cpu(), want)
    other = clip(8, as_yuv420=True, out=buf)                     # `out` reused; another seed draws other planes in 'random' mode
    assert other.data_ptr() == buf.data_ptr()
    assert torch.equal(other.cpu(), want) == (mode == "const")


# ------------------------------------------------------------------------------------------------ driver
def _model(which):
    if which == "head_sr":
        return _head_sr()[0]
    if which == "torso_sr":
        return _torso_sr()[0]
    return build_model(scn.Scene(H=64, W=64, T=2, torso=which == "torso", max_steps=16))


def _batch(m, which, T):
    H = R if which in ("head_sr", "torso_sr") else 64
    sc = scn.Scene(H=H, W=H, T=T, torso=which in ("torso", "torso_sr"), max_steps=16)
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"].cuda() for f in fis], "rays_d": [f["rays_d"].cuda() for f in fis],
            "poses": [f["poses"].cuda() for f in fis], "cond_wins": [scn.cond_window(sc.cond, t, m.smo_win_size).cuda() for t in range(T)],
            "bg_coords": sc.bg_coords.cuda(), "bg_img": sc.bg_color.reshape(1, -1, 3).cuda(),
            "eye_area_percent": (0.3 + 0.05 * torch.arange(T, dtype=torch.float32)).reshape(T, 1).cuda(), "lm68": scn.lm68_sequence(T).cuda()}


@pytest.mark.parametrize("which", ["head", "torso", "head_sr", "torso_sr"])
def test_driver_yuv420_batch_and_stream_equal_the_uint8_frames(which):
    m = _model(which)
    mode = "const"
    if which in ("head_sr", "torso_sr"):
        _noisy(m)
        mode = "random"
    T = 11
    batch = _batch(m, which, T)
    kw = {"T_thresh": 0.01, "sr_noise_mode": mode, "frames_per_call": 4}
    torch.manual_seed(3)
    u8 = driver.render_driver_batch(m, batch, as_uint8=True, **kw)
    H, W = u8.shape[1:3]
    want = _ref(u8, H, W)
    torch.manual_seed(3)
    whole = driver.render_driver_batch(m, batch, as_yuv420=True, **kw)
    assert whole.shape == (T, H * W * 3 // 2) and whole.dtype == torch.uint8 and whole.is_cuda
    assert torch.equal(whole.cpu(), want)
    torch.manual_seed(3)
    chunks = []
    for c in driver.iter_video_frames(m, batch, as_yuv420=True, **kw):
        assert c.device.type == "cpu" and c.is_pinned() and c.dtype == torch.uint8
        chunks.append(c.clone())
    assert [tuple(c.shape) for c in chunks] == [(4, H * W * 3 // 2), (4, H * W * 3 // 2), (3, H * W * 3 // 2)]
    assert torch.equal(torch.cat(chunks), want)
