"""genefaceplusplus_b200/driver.py with the SR checkpoints, on CPU: render_driver_batch hands every libgfpp stage of RADNeRFwithSR /
RADNeRFTorsowithSR the right chunk of the driver's batch (the stages are stubbed: they need the GPU), and iter_video_frames yields
the frames in order and waits for its streams when it is closed (streams and events stubbed as well)."""
import contextlib
import itertools

import pytest
import torch

from genefaceplusplus_b200 import driver
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR, RADNeRFwithSR

T = 9
R = 256


def _value(t):
    return (t + 1) / 16.0          # frame t's colour in the stubs: exact in fp32, and int(v * 255) is distinct per frame


def _batch(torso):
    """The dict prepare_batch_from_inp + forward_audio2secc build (genefacepp_infer.py:203-269, 400-429) for a T-frame clip."""
    sc = scn.Scene(H=R, W=R, T=T, torso=torso)
    fis = [sc.frame_inputs(t) for t in range(T)]
    return {"rays_o": [f["rays_o"] for f in fis], "rays_d": [f["rays_d"] for f in fis], "poses": [f["poses"] for f in fis],
            "cond_wins": [scn.cond_window(sc.cond, t) for t in range(T)], "bg_coords": sc.bg_coords, "bg_img": sc.bg_color.reshape(1, -1, 3),
            "eye_area_percent": torch.linspace(0.1, 0.9, T).reshape(T, 1), "lm68": scn.lm68_sequence(T)}


def _stub(m, batch, calls):
    """Stub the three libgfpp stages; each checks what it is handed and passes the frame identity on through the colour."""
    N = R * R

    def frames_of(rays_o):
        return [next(i for i in range(T) if torch.equal(rays_o[j], batch["rays_o"][i].reshape(N, 3))) for j in range(rays_o.shape[0])]

    def render_frames(cond_feat, **kw):
        idx = frames_of(kw["rays_o"])
        assert idx == list(range(idx[0], idx[0] + len(idx)))
        for j, i in enumerate(idx):
            assert torch.equal(kw["rays_d"][j], batch["rays_d"][i].reshape(N, 3))
        assert kw["rays_o"].shape == (len(idx), N, 3) and kw.get("pose6") is None and kw.get("bg_coords") is None
        calls.append(("nerf", idx, cond_feat.clone(), kw["bg_color"], kw["T_thresh"], kw["max_steps"]))
        rgb = torch.stack([torch.full((N, 3), _value(i)) for i in idx])
        if "u8_out" in kw:
            kw["u8_out"].copy_((rgb * 255).to(torch.uint8))
        return {"rgb_map": rgb, "weights_sum": torch.full((len(idx), N), 0.25)}

    def torso_composite_native(image, weights_sum, lm68, bg_coords, bg_color=None, want_maps=True, rgb_out=None):
        idx = [int(round(float(image[j, 0, 0]) * 16)) - 1 for j in range(image.shape[0])]
        assert torch.equal(weights_sum, torch.full_like(weights_sum, 0.25)) and not want_maps
        calls.append(("torso", idx, lm68.clone(), bg_coords, bg_color))
        return {"rgb_map": image}

    def forward_native(rgb_flat, noise_mode="random", clamp=False, out=None, frames_per_call=8, noise_planes=None, u8_out=None):
        n = rgb_flat.shape[0]
        assert rgb_flat.shape == (n, N, 3) and clamp and n <= frames_per_call <= driver.SR_FRAMES_PER_CALL
        assert out is not None or u8_out is not None
        idx = [int(round(float(rgb_flat[j, 0, 0]) * 16)) - 1 for j in range(n)]
        calls.append(("sr", idx, noise_mode, out is not None, u8_out is not None))
        for j, i in enumerate(idx):
            if out is not None:
                out[j] = _value(i)
            if u8_out is not None:
                u8_out[j] = i + 1

    m.render_frames = render_frames
    if isinstance(m, RADNeRFTorsowithSR):
        m.torso_composite_native = torso_composite_native
    m.sr_net.forward_native = forward_native


def _model(cls):
    hp = may_hparams(with_sr=True, add_eye_blink_cond=True, eye_blink_dim=2)
    return cls(hp).eval()


@pytest.mark.parametrize("as_uint8", [False, True])
@pytest.mark.parametrize("cls", [RADNeRFwithSR, RADNeRFTorsowithSR], ids=lambda c: c.__name__)
def test_render_driver_batch_sr_chunks(cls, as_uint8):
    m = _model(cls)
    torso = cls is RADNeRFTorsowithSR
    batch = _batch(torso)
    calls = []
    _stub(m, batch, calls)
    with torch.no_grad():
        feat = driver.cond_feat_from_windows(m, batch["cond_wins"], batch["eye_area_percent"])
        no_eye = driver.cond_feat_from_windows(m, batch["cond_wins"], None)
        for t in (0, T - 1):   # each row is the frame's own conditioning, eye value included
            one = m.cal_cond_feat(batch["cond_wins"][t], eye_area_percent=batch["eye_area_percent"][t])
            assert (feat[t] - one.reshape(-1)).abs().max().item() < 1e-6
    assert not torch.equal(feat, no_eye)
    out = driver.render_driver_batch(m, batch, T_thresh=0.02, frames_per_call=4, as_uint8=as_uint8, sr_noise_mode="const")
    chunks = [[0, 1, 2, 3], [4, 5, 6, 7], [8]]
    stages = ["nerf", "torso", "sr"] if torso else ["nerf", "sr"]
    assert [c[0] for c in calls] == stages * 3 and [c[1] for c in calls] == [ch for ch in chunks for _ in stages]
    for c in calls:
        s, e = c[1][0], c[1][-1] + 1
        if c[0] == "nerf":
            assert torch.equal(c[2], feat[s:e]) and c[4] == 0.02 and c[5] == m.hparams["max_steps"]
            # the torso-SR head field renders over a zero background (premultiplied colour); the head-SR one over bg_img
            assert torch.equal(c[3], torch.zeros(R * R, 3)) if torso else c[3] is batch["bg_img"]
        elif c[0] == "torso":
            assert torch.equal(c[2], batch["lm68"][s:e]) and c[3] is batch["bg_coords"] and c[4] is batch["bg_img"]
        else:
            assert c[2] == "const" and c[3] == (not as_uint8) and c[4] == as_uint8
    if as_uint8:
        assert out.dtype == torch.uint8 and out.shape == (T, 2 * R, 2 * R, 3)
        assert [int(out[t, 5, 7, 1]) for t in range(T)] == [t + 1 for t in range(T)]
    else:
        assert out.dtype == torch.float32 and out.shape == (T, 3, 2 * R, 2 * R)
        assert [float(out[t, 1, 5, 7]) for t in range(T)] == [_value(t) for t in range(T)]
    calls.clear()
    driver.render_driver_batch(m, batch, frames_per_call=32)
    assert [len(c[1]) for c in calls if c[0] == "sr"] == [8, 1]          # SR chunks of at most 8 frames


class _Stream:
    def __init__(self, log, name):
        self.log, self.name = log, name

    def wait_event(self, ev):
        self.log.append(("wait", self.name, ev.name))

    def synchronize(self):
        self.log.append(("sync", self.name))


def _fake_cuda(monkeypatch, log):
    names = itertools.cycle(["rendered0", "rendered1", "copied0", "copied1"])     # creation order in iter_video_frames

    class _Event:
        def __init__(self):
            self.name = next(names)

        def record(self, stream):
            log.append(("record", stream.name, self.name))

        def synchronize(self):
            log.append(("host_wait", self.name))

    compute = _Stream(log, "compute")
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: compute)
    monkeypatch.setattr(torch.cuda, "Stream", lambda device=None: _Stream(log, "side"))
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(driver, "_pinned", lambda shape: torch.empty(shape, dtype=torch.uint8))


@pytest.mark.parametrize("cls", [RADNeRFwithSR, RADNeRFTorsowithSR], ids=lambda c: c.__name__)
def test_iter_video_frames_order_and_close(cls, monkeypatch):
    m = _model(cls)
    batch = _batch(cls is RADNeRFTorsowithSR)
    calls, log = [], []
    _stub(m, batch, calls)
    _fake_cuda(monkeypatch, log)
    whole = driver.render_driver_batch(m, batch, frames_per_call=4, as_uint8=True, sr_noise_mode="none")
    got = [c.clone() for c in driver.iter_video_frames(m, batch, frames_per_call=4, sr_noise_mode="none")]
    assert [c.shape[0] for c in got] == [4, 4, 1] and torch.equal(torch.cat(got), whole)
    assert log[-2:] == [("sync", "side"), ("sync", "compute")]
    # chunk k+1 is queued before the host waits for chunk k's copy; buffer b is rendered into only after its last copy left it
    assert log.index(("record", "compute", "rendered1")) < log.index(("host_wait", "copied0"))
    assert [e for e in log if e[0] == "wait" and e[1] == "compute"] == [("wait", "compute", f"copied{k % 2}") for k in range(3)]

    # closed after the first chunk: the two queued chunks are all that was rendered, and both streams are waited for
    calls.clear()
    log.clear()
    gen = driver.iter_video_frames(m, batch, frames_per_call=4, sr_noise_mode="none")
    first = next(gen)
    assert first.shape == (4, 2 * R, 2 * R, 3) and [int(first[j, 0, 0, 0]) for j in range(4)] == [1, 2, 3, 4]
    gen.close()
    assert [c[1] for c in calls if c[0] == "sr"] == [[0, 1, 2, 3], [4, 5, 6, 7]]
    assert log[-2:] == [("sync", "side"), ("sync", "compute")]


def test_iter_video_frames_plain_torso_model(monkeypatch):
    """The non-SR classes stream the epilogue kernel's uint8 frames (render_frames' u8_out) through the same buffers."""
    hp = may_hparams()
    sc = scn.Scene(H=8, W=8, T=7, torso=True)
    m = RADNeRFTorso(hp).eval()
    m.load_state_dict(sc.state, strict=False)
    seen = []

    def render_frames(cond_feat, **kw):
        n = cond_feat.shape[0]
        seen.append((n, tuple(kw["pose6"].shape), "u8_out" in kw))
        if kw.get("u8_out") is not None:     # frame j of call c: value 10 c + j
            u8 = kw["u8_out"]
            u8.copy_((torch.arange(n, dtype=torch.uint8) + 10 * (len(seen) - 1)).view(n, 1, 1, 1).expand_as(u8))
        return {"rgb_map": torch.full((n, 64, 3), 0.5)}

    m.render_frames = render_frames
    fis = [sc.frame_inputs(t) for t in range(7)]
    batch = {"rays_o": [f["rays_o"] for f in fis], "rays_d": [f["rays_d"] for f in fis], "cond_wins": [scn.cond_window(sc.cond, t) for t in range(7)],
             "poses": [f["poses"] for f in fis], "bg_coords": sc.bg_coords, "bg_img": sc.bg_color}
    log = []
    _fake_cuda(monkeypatch, log)
    got = list(c.clone() for c in driver.iter_video_frames(m, batch, frames_per_call=3))
    assert [tuple(c.shape) for c in got] == [(3, 8, 8, 3), (3, 8, 8, 3), (1, 8, 8, 3)]
    assert seen == [(3, (3, 6), True), (3, (3, 6), True), (1, (1, 6), True)]
    assert [int(c[j, 0, 0, 0]) for c in got for j in range(c.shape[0])] == [0, 1, 2, 10, 11, 12, 20]
    assert log[-2:] == [("sync", "side"), ("sync", "compute")]


def test_sr_render_clip_as_uint8_on_the_torch_path(monkeypatch):
    """RADNeRFwithSR.render_clip(as_uint8=True) on CPU tensors (the NeRF clip stubbed: GPU): the video frames of the fp32 clip,
    HWC, written into a preallocated `out`; the NeRF clip is asked for fp32 frames."""
    from genefaceplusplus_b200.dist import to_uint8
    from genefaceplusplus_b200.renderer import RADNeRF
    m = RADNeRFwithSR(may_hparams(with_sr=True)).eval()
    fake = torch.rand(3, R * R, 3, generator=torch.Generator().manual_seed(0))
    asked = []
    monkeypatch.setattr(RADNeRF, "render_clip", lambda self, *a, **k: (asked.append(k), fake.clone())[1])
    args = (torch.eye(4).repeat(3, 1, 1), None, R, R)
    f32 = m.render_clip(*args, sr_noise_mode="none", sr_frames_per_call=2)
    buf = torch.zeros(3, 2 * R, 2 * R, 3, dtype=torch.uint8)
    u8 = m.render_clip(*args, sr_noise_mode="none", sr_frames_per_call=2, as_uint8=True, out=buf)
    assert u8 is buf and torch.equal(buf, to_uint8(f32.permute(0, 2, 3, 1)))
    assert all("as_uint8" not in k and "out" not in k for k in asked)
    with pytest.raises(ValueError):
        m.render_clip(*args, sr_noise_mode="none", as_uint8=True, out=torch.zeros(3, 3, 2 * R, 2 * R, dtype=torch.uint8))
