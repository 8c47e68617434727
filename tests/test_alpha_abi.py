"""Alpha-matte frames of the fused renderer (gfpp_outputs.alpha_map / rgba_u8, render_frames' alpha_out / rgba_out, the as_rgba
clip and driver APIs) without a GPU: the C-ABI mirror, every argument check (they all raise before anything is launched), what the
clip and driver APIs hand render_frames, and the epilogue kernels' register budget (nvcc cross-compiles)."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest
import torch

from genefaceplusplus_b200 import _capi, build, driver
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso, RADNeRFTorsowithSR, RADNeRFwithSR

MODEL_MAGIC = 0x67667070      # what gfpp_model_pack writes first ("gfpp")
P = ctypes.c_void_p
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gfpp.h")


# ------------------------------------------------------------------------------------------------ C-ABI
def test_outputs_mirror_appends_the_matte_fields():
    names = [f[0] for f in _capi.Outputs._fields_]
    assert names == ["rgb_map", "depth_map", "weights_sum", "torso_alpha_map", "torso_rgb_map", "torso_deform", "stats", "rgb_u8",
                     "alpha_map", "rgba_u8"]
    # every field that existed before keeps its offset: eight pointers, then the two new ones
    assert [getattr(_capi.Outputs, n).offset for n in names] == [8 * i for i in range(10)]
    assert ctypes.sizeof(_capi.Outputs) == 80
    body = open(HEADER).read().split("} gfpp_outputs;")[0].rsplit("typedef struct {", 1)[1]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\*\s*(\w+)\s*;", body) == names


def _frames(n_frames=2, n_rays=64):
    fr = _capi.Frames()
    fr.n_frames, fr.n_rays = n_frames, n_rays
    fr.rays_o, fr.rays_d, fr.cond_feat = 4096, 8192, 12288
    fr.max_steps = 16
    return fr


def _render(L, model, out, ws_bytes=1):
    return L.gfpp_render_frames(ctypes.byref(model), ctypes.byref(_frames()), ctypes.byref(out), P(4096), ws_bytes, None)


def test_render_frames_takes_rgba_alone_and_checks_its_alignment():
    L = _capi.lib()
    m = _capi.Model()
    m.opaque[0] = MODEL_MAGIC
    out = _capi.Outputs()
    assert _render(L, m, out) == -1
    assert L.gfpp_last_error() == b"render_frames: rgb_map (or rgb_u8) and cond_feat are required"
    out.alpha_map = 4096                      # the coverage alone is not a frame
    assert _render(L, m, out) == -1 and b"rgb_map (or rgb_u8)" in L.gfpp_last_error()
    out.rgba_u8 = 4098
    assert _render(L, m, out) == -1 and b"rgba_u8 must be 4-byte aligned" in L.gfpp_last_error()
    # a 4-byte aligned rgba_u8 alone passes every argument check: the workspace check is the last one before the launches
    out.alpha_map, out.rgba_u8 = None, 4100
    assert _render(L, m, out) == -3 and b"workspace too small" in L.gfpp_last_error()


# ------------------------------------------------------------------------------------------------ render_frames
def _cpu_model(cls=RADNeRF, torso=False, H=8, W=8):
    sc = scn.Scene(H=H, W=W, T=4, torso=torso)
    m = cls(sc.hparams).eval()
    m.load_state_dict(sc.state, strict=True)
    return m, sc


def _frames_kw(sc, n=2):
    fis = [sc.frame_inputs(t) for t in range(n)]
    kw = dict(rays_o=torch.cat([f["rays_o"] for f in fis]), rays_d=torch.cat([f["rays_d"] for f in fis]))
    if sc.torso:
        kw.update(pose6=torch.cat([f["poses"] for f in fis]), bg_coords=sc.bg_coords)
    return kw


@pytest.mark.parametrize("torso", [False, True], ids=["head", "torso"])
def test_render_frames_validates_the_matte_buffers(torso):
    m, sc = _cpu_model(RADNeRFTorso if torso else RADNeRF, torso)
    feat = torch.zeros(2, 64)
    kw = _frames_kw(sc)
    N = sc.H * sc.W
    u8 = torch.zeros(2 * N * 4 + 4, dtype=torch.uint8)
    bad_rgba = {
        "dtype": torch.zeros(2, N, 4),
        "shape": torch.zeros(2, N, 3, dtype=torch.uint8),
        "contiguity": torch.zeros(2, 4, N, dtype=torch.uint8).transpose(1, 2),
        "alignment": u8[1:1 + 2 * N * 4].view(2, N, 4),
        "device": torch.empty(2, N, 4, dtype=torch.uint8, device="meta"),
    }
    for what, t in bad_rgba.items():
        with pytest.raises(ValueError, match="rgba_out"):
            m.render_frames(feat, rgba_out=t, **kw)
    bad_alpha = {
        "dtype": torch.zeros(2, N, dtype=torch.float64),
        "shape": torch.zeros(2, N, 4),
        "contiguity": torch.zeros(N, 2).t(),
        "device": torch.empty(2, N, device="meta"),
    }
    for what, t in bad_alpha.items():
        with pytest.raises(ValueError, match="alpha_out"):
            m.render_frames(feat, alpha_out=t, rgba_out=u8[:2 * N * 4].view(2, N, 4), **kw)
    # well-formed buffers (rgba_out alone, or with alpha_out and a [F,H,W,4] view) get as far as the device check: no CPU path
    for extra in ({}, {"alpha_out": torch.zeros(2, N)}):
        with pytest.raises(_capi.GfppError, match="no CPU path"):
            m.render_frames(feat, rgba_out=u8[4:].view(2, sc.H, sc.W, 4), **extra, **kw)


# ------------------------------------------------------------------------------------------------ render_clip
def test_render_clip_as_rgba_arguments():
    m, sc = _cpu_model(RADNeRFTorso, True)
    poses = torch.stack([sc.pose(t) for t in range(3)])
    feat = torch.zeros(3, 64)
    N = sc.H * sc.W
    with pytest.raises(ValueError, match="background"):
        m.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=feat, bg_coords=sc.bg_coords, bg_color=sc.bg_color, as_rgba=True)
    with pytest.raises(ValueError, match="as_uint8"):
        m.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=feat, bg_coords=sc.bg_coords, as_rgba=True, as_uint8=True)
    for bad in (torch.zeros(3, N, 3, dtype=torch.uint8), torch.zeros(3, N, 4), torch.zeros(3, 4, N, dtype=torch.uint8).transpose(1, 2)):
        with pytest.raises(ValueError, match="out must be"):
            m.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=feat, bg_coords=sc.bg_coords, as_rgba=True, out=bad)

    calls = []

    def render_frames(cond_feat, **kw):
        calls.append((cond_feat.shape[0], sorted(k for k in ("rgb_out", "u8_out", "rgba_out") if k in kw), kw["bg_color"]))
        kw["rgba_out"].fill_(len(calls))
        return {"rgba_u8": kw["rgba_out"]}

    m.render_frames = render_frames
    buf = torch.zeros(3, sc.H, sc.W, 4, dtype=torch.uint8)
    got = m.render_clip(poses, sc.intrinsics, sc.H, sc.W, cond_feat=feat, bg_coords=sc.bg_coords, as_rgba=True, out=buf, frames_per_call=2)
    assert got.shape == (3, N, 4) and got.data_ptr() == buf.data_ptr()
    assert calls == [(2, ["rgba_out"], None), (1, ["rgba_out"], None)]
    assert got[:2].eq(1).all() and got[2].eq(2).all()


@pytest.mark.parametrize("cls", [RADNeRFwithSR, RADNeRFTorsowithSR], ids=lambda c: c.__name__)
def test_sr_models_have_no_rgba_clip(cls):
    m = cls(may_hparams(with_sr=True)).eval()
    with pytest.raises(ValueError, match="SR head is not linear"):
        m.render_clip(torch.eye(4).repeat(2, 1, 1), (1.0, 1.0, 128.0, 128.0), 256, 256, cond_feat=torch.zeros(2, 64), as_rgba=True)


# ------------------------------------------------------------------------------------------------ driver
def _batch(sc, T):
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"] for f in fis], "rays_d": [f["rays_d"] for f in fis], "poses": [f["poses"] for f in fis],
            "cond_wins": [scn.cond_window(sc.cond, t) for t in range(T)], "bg_coords": sc.bg_coords, "bg_img": sc.bg_color}


def test_render_driver_batch_as_rgba_hands_render_frames_the_matte_buffers():
    m, sc = _cpu_model(RADNeRFTorso, True)
    seen = []

    def render_frames(cond_feat, **kw):
        n = cond_feat.shape[0]
        seen.append((n, tuple(kw["rgba_out"].shape), kw["bg_color"], "u8_out" in kw or "rgb_out" in kw))
        kw["rgba_out"].copy_((torch.arange(n, dtype=torch.uint8) + 10 * (len(seen) - 1)).view(n, 1, 1).expand_as(kw["rgba_out"]))
        return {"rgba_u8": kw["rgba_out"]}

    m.render_frames = render_frames
    got = driver.render_driver_batch(m, _batch(sc, 4), frames_per_call=3, as_rgba=True)
    assert got.shape == (4, sc.H, sc.W, 4) and got.dtype == torch.uint8
    assert seen == [(3, (3, 64, 4), None, False), (1, (1, 64, 4), None, False)]
    assert [int(got[t, 0, 0, 0]) for t in range(4)] == [0, 1, 2, 10]


def test_driver_rejects_rgba_for_sr_models_and_with_uint8():
    m = RADNeRFwithSR(may_hparams(with_sr=True)).eval()
    batch = {"poses": [None] * 2}
    with pytest.raises(ValueError, match="SR head is not linear"):
        driver.render_driver_batch(m, batch, as_rgba=True)
    with pytest.raises(ValueError, match="SR head is not linear"):
        next(driver.iter_video_frames(m, batch, as_rgba=True))
    h, _ = _cpu_model()
    with pytest.raises(ValueError, match="as_uint8"):
        driver.render_driver_batch(h, batch, as_rgba=True, as_uint8=True)


# ------------------------------------------------------------------------------------------------ k_epilogue's budget
def test_epilogue_keeps_two_ctas_per_sm_without_spills():
    """k_epilogue and its matte-writing twin k_epilogue_matte (one body, the matte's stores a compile-time switch): both must stay at
    <= 128 registers (two CTAs of 256 threads per SM) with no spills."""
    with tempfile.TemporaryDirectory() as td:
        cmd = [build.NVCC, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "torso_kernel.cu"), "-o", os.path.join(td, "k.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cur, found = None, {}
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            k = re.search(r"\d(k_epilogue(?:_matte)?)E", m.group(1))
            cur = k.group(1) if k else None
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            found.setdefault(cur, {})["spills"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            found.setdefault(cur, {})["regs"] = int(m.group(1))
    print(f"registers and spill bytes: {found}")
    assert set(found) == {"k_epilogue", "k_epilogue_matte"}, r.stderr
    for k, v in found.items():
        assert v["spills"] == (0, 0) and v["regs"] * 256 * 2 <= 65536, (k, v)
