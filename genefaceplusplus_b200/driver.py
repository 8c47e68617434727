"""Driver-level shim (SURVEY.md 8(f) rank 1): the render loop of `GeneFace2Infer.forward_secc2video`
(inference/genefacepp_infer.py:433-486) without its T serial `render()` calls, per-frame `.cpu()` and fp32 frame stack.

`render_driver_batch` takes the very `batch` dict `prepare_batch_from_inp` builds (:203-269: lists `rays_o`, `rays_d`,
`cond_wins`, `poses`, `eye_area_percent`, plus `bg_coords`, `bg_img`) and returns the frames the driver would have produced,
rendering `frames_per_call` frames per libgfpp call with the conditioning nets batched over the clip.  The maintainer's
change in forward_secc2video is

    pred_rgbs = render_driver_batch(self.secc2video_model, batch, T_thresh=inp['raymarching_end_threshold'])   # [T,3,H,W] in [0,1], on the GPU
    out_imgs = video_uint8(pred_rgbs).cpu().numpy()                                                           # what imageio gets (:505)

For drivers that can hand over c2w poses instead of materialised rays (1.5 GB for 250 frames), `model.render_clip` generates
the rays in-kernel; this shim is for the unmodified batch layout.  All four model classes: for the `with_sr` checkpoints
(RADNeRFwithSR / RADNeRFTorsowithSR) the frames are the 512x512 `sr_rgb_map` the driver takes (:464-465, 480-481), and the
change is

    out_imgs = render_driver_batch(self.secc2video_model, batch, T_thresh=inp['raymarching_end_threshold'], as_uint8=True).cpu().numpy()

For the `low_memory_usage` mode (:449-470), `iter_video_frames` yields the frames as host uint8 chunks for `writer.append_data`,
with only two chunks of frames alive at any time.

With as_rgba=True both return alpha-matte frames [..,H,W,4] instead (non-SR models): premultiplied colour P and coverage A as
`(x*255).int()`, with no background in them (the batch's `bg_img` is not read), so that P + (1 - A) * B puts the head over any
background B, e.g. a different one per frame.

With as_yuv420=True both return the as_uint8 frames as planar I420 [.., H*W*3/2] (all four model classes; video.py), ready for
`ffmpeg -f rawvideo -pix_fmt yuv420p -s WxH -r 25 -i -` at half the bytes per frame.
"""
import torch

from . import video
from .dist import to_uint8
from .renderer import _no_sr_matte


def cond_feat_from_windows(model, cond_wins, eye_area_percent=None):
    """All frames' `cal_cond_feat` in one pass: cond_wins = list/stack of T windows [S,cond_win_size,C] (what the driver passes per frame,
    genefacepp_infer.py:420-422) -> [T,64].  Equals calling model.cal_cond_feat window by window."""
    wins = torch.stack([w.reshape(w.shape[0], -1) for w in cond_wins]) if not torch.is_tensor(cond_wins) else cond_wins.reshape(cond_wins.shape[0], cond_wins.shape[1], -1)
    T, S, C = wins.shape
    dev = model.density_bitfield.device
    wins = wins.to(dev).float()
    with torch.autocast(dev.type, enabled=False):
        feat = model.cond_prenet(wins.reshape(T * S, model.cond_win_size, C // model.cond_win_size))
        if model.add_eye_blink_cond:
            eye = None
            if eye_area_percent is not None and model.forwards_eye_area:
                eye = torch.as_tensor(eye_area_percent, dtype=torch.float32).reshape(T)
            feat = model._add_blink(feat, eye, T)
        feat = feat.view(T, S, -1)
        feat = model.cond_att_net.forward_batched(feat) if model.with_att else feat[:, S // 2]   # centre row, like cal_cond_feat_clip
    return feat


SR_FRAMES_PER_CALL = 8   # frames per SR-head call: its workspace is 68 MB per frame (as RADNeRF*withSR.render_clip)


def _is_sr(model):
    return hasattr(model, "sr_net")


def _frame_hw(model, batch):
    """(H, W) of the frames the driver writes: the NeRF image (H = W = sqrt(N)), or the SR head's 2x output."""
    if _is_sr(model):
        R = 2 * model.sr_input_resolution
        return R, R
    N = batch["rays_o"][0].numel() // 3
    H = int(round(N ** 0.5))
    return H, N // H


def _render_kw(model, T_thresh, dt_gamma, max_steps):
    hp = model.hparams
    return {"dt_gamma": hp["dt_gamma"] if dt_gamma is None else dt_gamma, "max_steps": hp["max_steps"] if max_steps is None else max_steps,
            "T_thresh": T_thresh}


def _check_formats(model, batch, as_uint8, as_rgba, as_yuv420):
    if as_rgba and as_uint8:
        raise ValueError("as_rgba and as_uint8 are two different frame formats: pick one")
    if as_yuv420 and (as_uint8 or as_rgba):
        raise ValueError("as_yuv420 is a frame format of its own: it cannot be combined with as_uint8 or as_rgba")
    _no_sr_matte(as_rgba and _is_sr(model))
    if as_yuv420:
        video.check_i420_size(*_frame_hw(model, batch))


def _render_chunk(model, batch, feat, s, e, kw, out=None, out_u8=None, out_rgba=None, sr_noise_mode="random"):
    """Frames [s, e) of the batch in one libgfpp call per stage.  Non-SR models: returns render_frames' result (`rgb_map` [n,N,3];
    with out_u8 [n,N,3] the uint8 frames go there instead; with out_rgba [n,N,4] the matte frames, without the background).
    SR models: the clamped 512x512 frames go into out [n,3,512,512] and/or out_u8 [n,512,512,3] -- what render()'s `sr_rgb_map`
    gives frame by frame: the head field with the frame's rays (torso-SR: on a zero background, then the torso field + composite
    with its `lm68` row over `bg_img`), then the SR head."""
    N = batch["rays_o"][0].numel() // 3
    rays_o = torch.stack([batch["rays_o"][i].reshape(N, 3) for i in range(s, e)])
    rays_d = torch.stack([batch["rays_d"][i].reshape(N, 3) for i in range(s, e)])
    if not _is_sr(model):
        pose6 = torch.stack([batch["poses"][i].reshape(6) for i in range(s, e)]) if model.has_torso else None
        bufs = {"rgba_out": out_rgba} if out_rgba is not None else {} if out_u8 is None else {"u8_out": out_u8}
        return model.render_frames(feat[s:e], rays_o=rays_o, rays_d=rays_d, pose6=pose6,
                                   bg_coords=batch["bg_coords"] if model.has_torso else None,
                                   bg_color=batch.get("bg_img") if out_rgba is None else None, **kw, want_torso_maps=False, **bufs)
    dev = model.density_bitfield.device
    with torch.autocast(dev.type, enabled=False):
        if hasattr(model, "torso_composite_native"):
            lm68 = torch.as_tensor(batch["lm68"]).reshape(-1, 136)[s:e]
            hd = model.render_frames(feat[s:e], rays_o=rays_o, rays_d=rays_d, bg_color=torch.zeros(N, 3, device=dev), **kw)
            img = model.torso_composite_native(hd["rgb_map"], hd["weights_sum"], lm68, batch["bg_coords"], batch.get("bg_img"),
                                               want_maps=False)["rgb_map"]
        else:
            img = model.render_frames(feat[s:e], rays_o=rays_o, rays_d=rays_d, bg_color=batch.get("bg_img"), **kw, want_aux=False)["rgb_map"]
        model.sr_net.forward_native(img, noise_mode=sr_noise_mode, clamp=True, out=out, u8_out=out_u8, frames_per_call=e - s)


def _render_chunk_i420(model, batch, feat, s, e, kw, H, W, out, sr_noise_mode):
    """Frames [s, e) as I420 into out [e-s, H*W*3/2]: _render_chunk's uint8 frames, written to the model's scratch buffer, converted."""
    frames = video.frame_scratch(model, (e - s, H, W, 3))
    _render_chunk(model, batch, feat, s, e, kw, out_u8=frames, sr_noise_mode=sr_noise_mode)
    video.rgb_u8_to_i420(frames, H, W, out=out)


@torch.no_grad()
def render_driver_batch(model, batch, T_thresh=1e-2, frames_per_call=32, dt_gamma=None, max_steps=None, as_uint8=False,
                        sr_noise_mode="random", as_rgba=False, as_yuv420=False):
    """-> [T,3,H,W] fp32 in [0,1] on the model's device (H = W = sqrt(N); SR models: the 512x512 `sr_rgb_map` frames), or with
    as_uint8 the video frames uint8 [T,H,W,3] `(rgb*255).int()`, written by the last kernel itself, or with as_rgba (non-SR models)
    the alpha-matte frames uint8 [T,H,W,4] of render_frames' rgba_out, or with as_yuv420 the as_uint8 frames as planar I420
    uint8 [T,H*W*3/2] (H and W even).  SR models take the batch's `lm68` [T,136] (torso-SR) and render at most SR_FRAMES_PER_CALL
    frames per call; sr_noise_mode as render()'s."""
    _check_formats(model, batch, as_uint8, as_rgba, as_yuv420)
    T = len(batch["poses"])
    dev = model.density_bitfield.device
    feat = cond_feat_from_windows(model, batch["cond_wins"], batch.get("eye_area_percent"))
    H, W = _frame_hw(model, batch)
    kw = _render_kw(model, T_thresh, dt_gamma, max_steps)
    if as_yuv420:
        fpc = min(frames_per_call, SR_FRAMES_PER_CALL) if _is_sr(model) else frames_per_call
        out = torch.empty(T, video.i420_frame_bytes(H, W), device=dev, dtype=torch.uint8)
        for s in range(0, T, fpc):
            e = min(T, s + fpc)
            _render_chunk_i420(model, batch, feat, s, e, kw, H, W, out[s:e], sr_noise_mode)
        return out
    if _is_sr(model):
        fpc = min(frames_per_call, SR_FRAMES_PER_CALL)
        out = torch.empty((T, H, W, 3) if as_uint8 else (T, 3, H, W), device=dev, dtype=torch.uint8 if as_uint8 else torch.float32)
        for s in range(0, T, fpc):
            e = min(T, s + fpc)
            _render_chunk(model, batch, feat, s, e, kw, out=None if as_uint8 else out[s:e], out_u8=out[s:e] if as_uint8 else None,
                          sr_noise_mode=sr_noise_mode)
        return out
    N = H * W
    C = 4 if as_rgba else 3
    out = torch.empty(T, N, C, device=dev, dtype=torch.uint8 if as_uint8 or as_rgba else torch.float32)
    for s in range(0, T, frames_per_call):
        e = min(T, s + frames_per_call)
        if as_rgba:
            _render_chunk(model, batch, feat, s, e, kw, out_rgba=out[s:e])
        elif as_uint8:
            _render_chunk(model, batch, feat, s, e, kw, out_u8=out[s:e])
        else:
            out[s:e] = _render_chunk(model, batch, feat, s, e, kw)["rgb_map"]
    return out.view(T, H, W, C) if as_uint8 or as_rgba else out.view(T, H, W, 3).permute(0, 3, 1, 2)


def _pinned(shape):
    return torch.empty(shape, dtype=torch.uint8, pin_memory=True)


@torch.no_grad()
def iter_video_frames(model, batch, frames_per_call=8, T_thresh=1e-2, dt_gamma=None, max_steps=None, sr_noise_mode="random",
                      as_rgba=False, as_yuv420=False):
    """The `low_memory_usage` loop of forward_secc2video (genefacepp_infer.py:449-470) for all four model classes: yields the
    clip's video frames -- what render_driver_batch(..., as_uint8=True) returns -- as host uint8 [n,H,W,3] chunks in frame order
    (n <= frames_per_call; SR models: <= SR_FRAMES_PER_CALL), e.g. `for c in iter_video_frames(...): for f in c.numpy(): writer.append_data(f)`.
    as_rgba (non-SR models): the alpha-matte frames of render_driver_batch(..., as_rgba=True) instead, as [n,H,W,4] chunks.
    as_yuv420: the I420 frames of render_driver_batch(..., as_yuv420=True), as [n,H*W*3/2] chunks, each one write to an ffmpeg
    rawvideo pipe (`proc.stdin.write(c.numpy().tobytes())`).

    Two device and two pinned host buffers: chunk k+1 renders on the current stream while chunk k is copied to the host on a
    side stream and handed to the caller.  A yielded chunk stays valid until the generator is advanced.  When the generator
    ends, fails or is closed early, it waits for both streams: no queued work is left behind."""
    _check_formats(model, batch, False, as_rgba, as_yuv420)
    T = len(batch["poses"])
    dev = model.density_bitfield.device
    feat = cond_feat_from_windows(model, batch["cond_wins"], batch.get("eye_area_percent"))
    H, W = _frame_hw(model, batch)
    kw = _render_kw(model, T_thresh, dt_gamma, max_steps)
    fpc = min(frames_per_call, SR_FRAMES_PER_CALL) if _is_sr(model) else frames_per_call
    starts = list(range(0, T, fpc))
    compute = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    rows = min(fpc, T)
    shape = (rows, video.i420_frame_bytes(H, W)) if as_yuv420 else (rows, H, W, 4 if as_rgba else 3)
    dbuf = [torch.empty(shape, device=dev, dtype=torch.uint8) for _ in range(2)]
    hbuf = [_pinned(shape) for _ in range(2)]
    rendered = [torch.cuda.Event() for _ in range(2)]
    copied = [torch.cuda.Event() for _ in range(2)]

    def launch(k):
        """Queue chunk k: render into device buffer k % 2, copy it to host buffer k % 2 on the side stream."""
        s, b = starts[k], k % 2
        e = min(T, s + fpc)
        compute.wait_event(copied[b])           # chunk k-2 has left device buffer b
        if as_yuv420:
            _render_chunk_i420(model, batch, feat, s, e, kw, H, W, dbuf[b][:e - s], sr_noise_mode)
        else:
            dst = {"out_rgba": dbuf[b][:e - s]} if as_rgba else {"out_u8": dbuf[b][:e - s]}
            _render_chunk(model, batch, feat, s, e, kw, sr_noise_mode=sr_noise_mode, **dst)
        rendered[b].record(compute)
        side.wait_event(rendered[b])
        with torch.cuda.stream(side):
            hbuf[b][:e - s].copy_(dbuf[b][:e - s], non_blocking=True)
        copied[b].record(side)
        return e - s

    try:
        n = launch(0) if starts else 0
        for k in range(len(starts)):
            n_next = launch(k + 1) if k + 1 < len(starts) else 0   # host buffer (k+1) % 2 was handed out as chunk k-1: released
            copied[k % 2].synchronize()
            yield hbuf[k % 2][:n]
            n = n_next
    finally:
        side.synchronize()
        compute.synchronize()


def video_uint8(pred_rgbs):
    """[T,3,H,W] in [0,1] -> uint8 [T,H,W,3]: the driver's `((x*2-1).clamp(-1,1) + 1)/2 * 255 -> int` (:488-505) in one step."""
    return to_uint8(pred_rgbs.permute(0, 2, 3, 1))
