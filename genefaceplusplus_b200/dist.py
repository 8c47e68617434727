"""Frame-parallel multi-GPU rendering (SURVEY.md 8(e)).

Frames of a clip are independent units: rank r of G renders the contiguous block
`frames[r*T/G : (r+1)*T/G]` (weights and tables, 29.7 MB, are replicated), then ONE collective at the
end gathers the rendered RGB of every rank so that each rank (or just rank 0) holds the whole clip in
video order.  There is no other exchange: the reference's inference path has no multi-GPU mode at all
(inference/genefacepp_infer.py:474-486 is a serial loop on one GPU).

The collective is `torch.distributed.all_gather_into_tensor` (NCCL on GPUs; gloo on CPU for the tests).
"""
import torch
import torch.distributed as dist


def frame_block(T: int, rank: int, world: int):
    """Contiguous, balanced partition of T frames; the first T % world ranks get one extra frame."""
    base, extra = divmod(T, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def padded_block_len(T: int, world: int) -> int:
    return (T + world - 1) // world


def gather_frames(local: torch.Tensor, T: int, group=None) -> torch.Tensor:
    """All-gather per-rank frame blocks [t_r, ...] into the full clip [T, ...] in video order.

    Blocks are padded to the common length ceil(T/world) so that a single all_gather_into_tensor
    moves everything; the padding rows are dropped afterwards."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    blk = padded_block_len(T, world)
    s, e = frame_block(T, rank, world)
    assert local.shape[0] == e - s, (local.shape, s, e)
    if local.shape[0] != blk:
        pad = torch.zeros((blk - local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        local = torch.cat([local, pad], 0)
    local = local.contiguous()
    full = torch.empty((world * blk,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(full, local, group=group)
    pieces = []
    for r in range(world):
        rs, re = frame_block(T, r, world)
        pieces.append(full[r * blk: r * blk + (re - rs)])
    return torch.cat(pieces, 0) if any(p.shape[0] != blk for p in pieces) else full[: T]


class OverlappedGather:
    """All-gather of a clip in CHUNKS, overlapped with rendering: while the kernels of chunk k+1 run on the compute stream, the
    uint8 frames of chunk k travel over NVLink on the collective's own stream (`all_gather_into_tensor(async_op=True)`, the same
    collective `gather_frames` uses).  Every rank renders the same number of frames `t_local` (weak scaling; pad the clip
    otherwise).  Each chunk lands in a staging slab [world, chunk, ...]; `finish()` waits for the collectives and moves the slabs
    into video order (one device-side copy of the clip, ~1 ms for 1.5 GB).  Usage:

        og = OverlappedGather(t_local, frame_shape, dtype, device)       # once; owns staging + result buffers
        for a, b in chunks: render frames [a, b) into local[a:b]; og.push(local, a, b)
        full = og.finish()                                               # [world * t_local, ...] in video order
    """

    def __init__(self, t_local, frame_shape, dtype, device, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.full = torch.empty((self.world, t_local) + tuple(frame_shape), dtype=dtype, device=device)
        self.stage = torch.empty((self.world * t_local,) + tuple(frame_shape), dtype=dtype, device=device) if self.world > 1 else None
        self.t_local = t_local
        self.work = []          # (work handle, a, b)

    def push(self, local, a, b):
        if self.world == 1:
            self.full[0, a:b].copy_(local[a:b])
            return
        # staging slab of this chunk: rows [world * a, world * b) viewed as [world, b - a, ...]; NCCL's stream waits on the current
        # (compute) stream, so the chunk is complete before the collective reads it
        slab = self.stage[self.world * a: self.world * b]
        self.work.append((dist.all_gather_into_tensor(slab, local[a:b].contiguous(), group=self.group, async_op=True), a, b))

    def finish(self):
        for w, a, b in self.work:
            w.wait()                                                 # makes the current stream wait for the collective
            slab = self.stage[self.world * a: self.world * b].view((self.world, b - a) + tuple(self.full.shape[2:]))
            self.full[:, a:b].copy_(slab)
        self.work = []
        return self.full.view((self.world * self.t_local,) + tuple(self.full.shape[2:]))


def to_uint8(rgb: torch.Tensor) -> torch.Tensor:
    """(x * 255).int() -> uint8, exactly what the driver writes to the video (genefacepp_infer.py:469, 505)."""
    return (rgb * 255.0).to(torch.int32).clamp_(0, 255).to(torch.uint8)


def render_clip_sharded(model, poses_c2w, intrinsics, H, W, cond_seq, *, bg_color=None, bg_coords=None, T_thresh=1e-2,
                        frames_per_call=64, as_uint8=False, gather=True, group=None, eye_area_percent=None, lm68_seq=None, **render_kw):
    """Render this rank's block of the clip with `model.render_clip` and all-gather the result.

    `cond_seq` (and `eye_area_percent` [T] for the blink-conditioned models) is the FULL sequence on every rank -- the +-2-frame
    smoothing window needs its halo; it is tiny -- so conditioning features at block edges equal the single-GPU ones.  Per-frame
    inputs of the SR models (`lm68_seq` [T,136]) are sliced to the rank's block; `render_kw` goes to `render_clip` unchanged
    (`sr_noise_mode=...`).  Works for all four model classes: [T,N,3] frames for the plain models, [T,3,512,512] for the SR ones.
    The I420 frames of render_clip(as_yuv420=True) are not offered here: convert gathered uint8 frames with video.rgb_u8_to_i420."""
    if render_kw.get("as_yuv420"):
        raise ValueError("render_clip_sharded does not produce I420 frames: convert gathered uint8 frames with video.rgb_u8_to_i420")
    T = poses_c2w.shape[0]
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank(group) if world > 1 else 0
    s, e = frame_block(T, rank, world)
    cond_seq = cond_seq.to(model.density_bitfield.device)
    cond_feat = (model.cal_cond_feat_clip(cond_seq) if eye_area_percent is None else model.cal_cond_feat_clip(cond_seq, eye_area_percent=eye_area_percent))[s:e]
    kw = dict(cond_feat=cond_feat, bg_color=bg_color, bg_coords=bg_coords, T_thresh=T_thresh, frames_per_call=frames_per_call, **render_kw)
    if lm68_seq is not None:
        kw["lm68_seq"] = lm68_seq[s:e]
    local = model.render_clip(poses_c2w[s:e], intrinsics, H, W, **kw)
    if as_uint8:
        local = to_uint8(local)
    return gather_frames(local, T, group) if gather else local
