"""Planar I420 video frames (gfpp.h section N, video.py, the as_yuv420 clip and driver APIs) without a GPU: the C-ABI and its
ctypes mirror, every argument check (all of them fail before any CUDA call or device work), what the clip and driver APIs hand
render_frames and the converter, the numpy restatement against hand values, and the kernels' register budget (nvcc cross-compiles)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import _capi, build, driver, video
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso, RADNeRFTorsowithSR, RADNeRFwithSR

INVALID = -1
FAKE = 0x10000          # never dereferenced: validation fails first
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gfpp.h")


@pytest.fixture(scope="module")
def L():
    build.build()
    return _capi.lib()


# ------------------------------------------------------------------------------------------------ C-ABI
def test_symbol_and_ctypes_mirror(L):
    assert "gfpp_rgb_u8_to_i420" in _capi.EXPORTS and hasattr(L, "gfpp_rgb_u8_to_i420")
    P, u32 = ctypes.c_void_p, ctypes.c_uint32
    assert L.gfpp_rgb_u8_to_i420.argtypes == [P, u32, u32, u32, P, P]
    decl = re.search(r"GFPP_API int gfpp_rgb_u8_to_i420\(([^)]*)\);", open(HEADER).read())
    assert decl and [a.split()[-1].lstrip("*") for a in decl.group(1).split(",")] == ["rgb", "F", "H", "W", "out", "stream"]


def test_validation_before_any_cuda_call(L):
    def conv(rgb=FAKE, F=2, H=4, W=6, out=FAKE):
        return L.gfpp_rgb_u8_to_i420(rgb, F, H, W, out, None)

    launches = L.gfpp_last_launch_count()             # of this thread's last call that launched: a refusal leaves it alone
    cases = {
        "null pointer": [dict(rgb=None), dict(out=None)],
        "no frames": [dict(F=0)],
        "must be even": [dict(H=0), dict(W=0), dict(H=3), dict(W=5), dict(H=511, W=512), dict(H=512, W=511)],
        "overflow": [dict(F=2, H=1 << 31, W=1 << 31), dict(F=(1 << 32) - 2, H=1 << 16, W=1 << 16), dict(F=1 << 31, H=1 << 31, W=1 << 31)],
    }
    for what, args in cases.items():
        for a in args:
            assert conv(**a) == INVALID, (what, a)
            assert what.encode() in L.gfpp_last_error(), (what, a, L.gfpp_last_error())
    assert L.gfpp_last_launch_count() == launches


# ------------------------------------------------------------------------------------------------ the numpy restatement
def _literal(rgb):
    """The header's formulas pixel by pixel and block by block, in plain Python integers."""
    F, H, W, _ = rgb.shape
    out = np.zeros((F, H * W * 3 // 2), dtype=np.uint8)
    for f in range(F):
        for i in range(H):
            for j in range(W):
                R, G, B = (int(c) for c in rgb[f, i, j])
                out[f, i * W + j] = ((66 * R + 129 * G + 25 * B + 128) >> 8) + 16
        for i in range(H // 2):
            for j in range(W // 2):
                R, G, B = ((sum(int(rgb[f, 2 * i + a, 2 * j + b, c]) for a in (0, 1) for b in (0, 1)) + 2) >> 2 for c in range(3))
                k = i * (W // 2) + j
                out[f, H * W + k] = ((-38 * R - 74 * G + 112 * B + 128) >> 8) + 128
                out[f, H * W + H * W // 4 + k] = ((112 * R - 94 * G - 18 * B + 128) >> 8) + 128
    return out


def _solid(r, g, b, H=2, W=4):
    return np.broadcast_to(np.array([r, g, b], dtype=np.uint8), (1, H, W, 3)).copy()


def test_reference_hand_values():
    def yuv(rgb):
        o = video.i420_reference(rgb)[0]
        return int(o[0]), int(o[8]), int(o[10])      # Y of pixel 0, U and V of block 0 (H=2, W=4: 8 luma, 2 + 2 chroma bytes)

    assert yuv(_solid(0, 0, 0)) == (16, 128, 128)                # black
    assert yuv(_solid(255, 255, 255)) == (235, 128, 128)         # white
    assert yuv(_solid(0, 0, 255))[1] == 240                      # U's extremes: pure blue, and yellow (-28432 >> 8 = -112)
    assert yuv(_solid(255, 255, 0))[1] == 16
    assert yuv(_solid(255, 0, 0))[2] == 240                      # V's extremes: pure red, and cyan
    assert yuv(_solid(0, 255, 255))[2] == 16
    # the block mean rounds half up: with R = G = 0, U is 129 from a blue mean of 2 and 128 from 1 (112 B + 128 crosses 256)
    for blues, u in (([0, 2, 2, 2], 129), ([1, 1, 1, 2], 128), ([2, 2, 2, 2], 129), ([1, 1, 1, 1], 128)):
        px = np.zeros((1, 2, 2, 3), dtype=np.uint8)
        px[0, :, :, 2] = np.array(blues, dtype=np.uint8).reshape(2, 2)
        assert int(video.i420_reference(px)[0, 4]) == u, blues
    assert video.i420_reference(_solid(7, 7, 7, H=4, W=6)).shape == (1, 36)


@pytest.mark.parametrize("F,H,W", [(1, 2, 2), (2, 4, 6), (1, 6, 10)])
def test_reference_equals_the_literal_formulas(F, H, W):
    rgb = np.random.default_rng(F * 100 + H * 10 + W).integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    rgb[0, 0, 0] = 0
    rgb[-1, -1, -1] = 255
    got = video.i420_reference(rgb)
    assert got.dtype == np.uint8 and got.shape == (F, H * W * 3 // 2)
    assert np.array_equal(got, _literal(rgb))
    assert got[:, : H * W].min() >= 16 and got[:, : H * W].max() <= 235 and got[:, H * W:].min() >= 16 and got[:, H * W:].max() <= 240


# ------------------------------------------------------------------------------------------------ Python guards
@pytest.fixture
def no_library(monkeypatch):
    monkeypatch.setattr(_capi, "lib", lambda: pytest.fail("the library was reached"))


def test_converter_guards(no_library):
    rgb = torch.zeros(2, 4, 6, 3, dtype=torch.uint8)
    for H, W in ((3, 6), (4, 5), (0, 6)):
        with pytest.raises(ValueError, match="even"):
            video.rgb_u8_to_i420(torch.zeros(2, H, W, 3, dtype=torch.uint8), H, W)
    with pytest.raises(ValueError, match="rgb must be"):
        video.rgb_u8_to_i420(rgb.float(), 4, 6)
    with pytest.raises(ValueError, match="rgb must be"):
        video.rgb_u8_to_i420(rgb[:, :3], 4, 6)
    for bad in (torch.zeros(2, 35, dtype=torch.uint8), torch.zeros(2, 36), torch.zeros(36, 2, dtype=torch.uint8).t(),
                torch.empty(2, 36, dtype=torch.uint8, device="meta")):
        with pytest.raises(ValueError, match="out must be"):
            video.rgb_u8_to_i420(rgb, 4, 6, out=bad)
    with pytest.raises(ValueError):
        video.i420_reference(np.zeros((1, 3, 4, 3), dtype=np.uint8))


def test_converter_has_no_cpu_path():
    with pytest.raises(_capi.GfppError, match="no CPU path"):
        video.rgb_u8_to_i420(torch.zeros(1, 2, 2, 3, dtype=torch.uint8), 2, 2)


def _cpu_model(cls=RADNeRFTorso, torso=True, H=8, W=8):
    sc = scn.Scene(H=H, W=W, T=4, torso=torso)
    m = cls(sc.hparams).eval()
    m.load_state_dict(sc.state, strict=True)
    return m, sc


@pytest.mark.parametrize("torso", [False, True], ids=["head", "torso"])
def test_render_clip_guards_precede_any_rendering(torso, no_library):
    m, sc = _cpu_model(RADNeRFTorso if torso else RADNeRF, torso)
    m.render_frames = lambda *a, **k: pytest.fail("render_frames was reached")
    poses = torch.stack([sc.pose(t) for t in range(3)])
    kw = dict(cond_feat=torch.zeros(3, 64), bg_coords=sc.bg_coords if torso else None)
    for other in ("as_uint8", "as_rgba"):
        with pytest.raises(ValueError, match="as_yuv420"):
            m.render_clip(poses, sc.intrinsics, sc.H, sc.W, as_yuv420=True, **{other: True}, **kw)
    for H, W in ((7, 8), (8, 7)):
        with pytest.raises(ValueError, match="even"):
            m.render_clip(poses, sc.intrinsics, H, W, as_yuv420=True, **kw)
    fb = sc.H * sc.W * 3 // 2
    for bad in (torch.zeros(3, fb + 1, dtype=torch.uint8), torch.zeros(3, sc.H * sc.W, 3, dtype=torch.uint8), torch.zeros(3, fb),
                torch.zeros(fb, 3, dtype=torch.uint8).t()):
        with pytest.raises(ValueError, match="out must be"):
            m.render_clip(poses, sc.intrinsics, sc.H, sc.W, as_yuv420=True, out=bad, **kw)


@pytest.mark.parametrize("cls", [RADNeRFwithSR, RADNeRFTorsowithSR], ids=lambda c: c.__name__)
def test_sr_render_clip_guards_precede_any_rendering(cls, no_library):
    m = cls(may_hparams(with_sr=True)).eval()
    m.render_frames = lambda *a, **k: pytest.fail("render_frames was reached")
    poses, kw = torch.eye(4).repeat(2, 1, 1), dict(cond_feat=torch.zeros(2, 64))
    with pytest.raises(ValueError, match="as_yuv420"):
        m.render_clip(poses, (1.0, 1.0, 128.0, 128.0), 256, 256, as_yuv420=True, as_uint8=True, **kw)
    for bad in (torch.zeros(2, 512 * 512 * 3, dtype=torch.uint8), torch.zeros(2, 512 * 512 * 3 // 2), torch.zeros(2, 512, 512, 3, dtype=torch.uint8)):
        with pytest.raises(ValueError, match="out must be"):
            m.render_clip(poses, (1.0, 1.0, 128.0, 128.0), 256, 256, as_yuv420=True, out=bad, **kw)


def _batch(sc, T):
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"] for f in fis], "rays_d": [f["rays_d"] for f in fis], "poses": [f["poses"] for f in fis],
            "cond_wins": [scn.cond_window(sc.cond, t) for t in range(T)], "bg_coords": sc.bg_coords, "bg_img": sc.bg_color}


def test_driver_guards_precede_any_device_work(monkeypatch, no_library):
    monkeypatch.setattr(driver, "cond_feat_from_windows", lambda *a, **k: pytest.fail("the conditioning nets were reached"))
    m, sc = _cpu_model()
    batch = _batch(sc, 2)
    for other in ("as_uint8", "as_rgba"):
        with pytest.raises(ValueError, match="as_yuv420"):
            driver.render_driver_batch(m, batch, as_yuv420=True, **{other: True})
    with pytest.raises(ValueError, match="as_yuv420"):
        next(driver.iter_video_frames(m, batch, as_yuv420=True, as_rgba=True))
    odd = dict(batch, rays_o=[torch.zeros(15 * 15, 3)] * 2)            # 15x15 frames
    with pytest.raises(ValueError, match="even"):
        driver.render_driver_batch(m, odd, as_yuv420=True)
    with pytest.raises(ValueError, match="even"):
        next(driver.iter_video_frames(m, odd, as_yuv420=True))


def test_sharded_clip_does_not_take_the_i420_flag():
    from genefaceplusplus_b200.dist import render_clip_sharded
    m, sc = _cpu_model()
    with pytest.raises(ValueError, match="I420"):
        render_clip_sharded(m, torch.eye(4).repeat(2, 1, 1), sc.intrinsics, sc.H, sc.W, sc.cond, as_yuv420=True)


# ------------------------------------------------------------------------------------------------ plumbing
def _host_converter(calls):
    def conv(rgb, H, W, out=None):
        calls.append((tuple(rgb.shape), H, W, out.data_ptr()))
        out.copy_(torch.from_numpy(video.i420_reference(rgb.reshape(-1, H, W, 3).numpy())).reshape(out.shape))
        return out
    return conv


def test_render_clip_hands_each_call_the_scratch_frames(monkeypatch):
    m, sc = _cpu_model(H=6, W=8)
    poses = torch.stack([sc.pose(t) for t in range(5)])
    N = sc.H * sc.W
    seen, conv = [], []
    want = []

    def render_frames(cond_feat, **kw):
        n = cond_feat.shape[0]
        seen.append((n, sorted(k for k in ("rgb_out", "u8_out", "rgba_out") if k in kw), kw["bg_color"] is not None))
        frames = torch.randint(0, 256, (n, N, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(len(seen)))
        kw["u8_out"].copy_(frames)
        want.append(frames)
        return {"rgb_u8": kw["u8_out"]}

    m.render_frames = render_frames
    monkeypatch.setattr(video, "rgb_u8_to_i420", _host_converter(conv))
    buf = torch.zeros(5, N * 3 // 2, dtype=torch.uint8)
    got = m.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=torch.zeros(5, 64), bg_coords=sc.bg_coords, bg_color=sc.bg_color,
                        as_yuv420=True, out=buf, frames_per_call=2)
    assert got.data_ptr() == buf.data_ptr() and got.shape == (5, N * 3 // 2) and got.dtype == torch.uint8
    assert seen == [(2, ["u8_out"], True), (2, ["u8_out"], True), (1, ["u8_out"], True)]
    assert [c[:3] for c in conv] == [((2, N, 3), sc.H, sc.W), ((2, N, 3), sc.H, sc.W), ((1, N, 3), sc.H, sc.W)]
    assert [c[3] for c in conv] == [buf[s].data_ptr() for s in (0, 2, 4)]
    ref = video.i420_reference(torch.cat(want).reshape(5, sc.H, sc.W, 3).numpy())
    assert np.array_equal(got.numpy(), ref)
    assert "_i420_scratch" in m.__dict__ and "_i420_scratch" not in m.state_dict()


def test_render_driver_batch_as_yuv420(monkeypatch):
    m, sc = _cpu_model()
    seen, conv = [], []

    def render_frames(cond_feat, **kw):
        n = cond_feat.shape[0]
        seen.append((n, tuple(kw["u8_out"].shape), "rgb_out" in kw or "rgba_out" in kw))
        kw["u8_out"].copy_((torch.arange(n, dtype=torch.uint8) * 40 + 10 * len(seen)).view(n, 1, 1, 1).expand_as(kw["u8_out"]))
        return {"rgb_u8": kw["u8_out"]}

    m.render_frames = render_frames
    monkeypatch.setattr(video, "rgb_u8_to_i420", _host_converter(conv))
    got = driver.render_driver_batch(m, _batch(sc, 4), frames_per_call=3, as_yuv420=True)
    assert got.shape == (4, sc.H * sc.W * 3 // 2) and got.dtype == torch.uint8
    assert seen == [(3, (3, sc.H, sc.W, 3), False), (1, (1, sc.H, sc.W, 3), False)]
    grey = [10, 50, 90, 20]                                   # every frame is one grey level: Y, U and V are constant per frame
    want = video.i420_reference(np.stack([_solid(g, g, g, sc.H, sc.W)[0] for g in grey]))
    assert np.array_equal(got.numpy(), want)


# ------------------------------------------------------------------------------------------------ the kernels' budget
def test_kernels_compile_spill_free_for_sm90a():
    cu = os.path.join(build.CSRC, "video_kernels.cu")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas=-v", "-c", cu, "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert len(entries) == 2 and all("k_rgb_u8_to_i420" in e for e in entries), r.stderr
    stacks = [ln for ln in r.stderr.splitlines() if "spill stores" in ln]
    assert len(stacks) == 2 and all("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in ln for ln in stacks), stacks
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", r.stderr)]
    print(f"k_rgb_u8_to_i420<4>, <2>: registers {regs}")
    assert len(regs) == 2 and max(regs) <= 64, regs
