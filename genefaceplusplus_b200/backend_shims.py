"""Level-B drop-in (SURVEY.md 8(b) "B-native"): register ctypes-backed modules under the names the reference's Python
imports its CUDA extensions by -- `_raymarching_face`, `_gridencoder`, `_shencoder`, `_freqencoder`
(modules/radnerfs/raymarching/raymarching.py:9-12, encoders/*/: `try: import _x as _backend`) -- so the UNMODIFIED reference
wrappers run on libgfpp's per-op kernels.  Call `install()` before `import modules.radnerfs`.

Inference exports: near_far_from_aabb, march_rays, composite_rays, grid_encode_forward, sh_encode_forward, freq_encode_forward.
Training-side exports (SURVEY.md 8(f) rank 4; csrc/train_kernels.cu): march_rays_train(+_backward), composite_rays_train_forward /
_backward, grid_encode_forward with dy_dx, grid_encode_backward, grad_total_variation, packbits, morton3D(+_invert, _dilation),
sph_from_ray -- fp32.  Under autocast the reference hands the grid encoder half tables (grid.py:41-44, C = 2): grid_encode_forward
and grid_encode_backward dispatch on the table's dtype like its AT_DISPATCH_FLOATING_TYPES_AND_HALF, fp32 to the fp32 ops of gfpp.h
sections (A) / (D), half to the half ops of section (L); a half table with fp32 outputs (or any other mix) raises RuntimeError, as the
reference's data_ptr<scalar_t>() does.  Every other op stays fp32 under autocast (custom_fwd(cast_inputs=torch.float32)).  The
input-gradient ops of the SH / frequency encoders (only needed when optimising camera poses through the view direction) still raise.
"""
import ctypes
import sys
import types

import numpy as np
import torch

from . import _capi


def _P(t, dtype=None):
    """Device pointer with the checks the reference's pybind layer makes (CHECK_CUDA / CHECK_CONTIGUOUS / dtype): a CPU, strided
    or wrongly typed tensor raises RuntimeError here instead of faulting asynchronously inside a kernel."""
    if not torch.is_tensor(t) or not t.is_cuda:
        raise RuntimeError("libgfpp: expected a CUDA tensor")
    if not t.is_contiguous():
        raise RuntimeError("libgfpp: expected a contiguous tensor")
    want = dtype if dtype is not None else _DTYPES.get(t.dtype)
    if want is None or t.dtype != want:
        raise RuntimeError(f"libgfpp: unsupported dtype {t.dtype} here (expected {want or 'fp32 / int32 / uint8'}; fp16 only for the grid encoder's half buffers)")
    return ctypes.c_void_p(t.data_ptr())


_DTYPES = {torch.float32: torch.float32, torch.int32: torch.int32, torch.uint8: torch.uint8}
_OFFSETS_HOST = {}


def _offsets_host(offsets):
    """Host copy of a grid's level offsets, cached per offsets TENSOR: no D2H sync per encoder call.  The cache entry holds a
    reference to the tensor, so its device address cannot be handed to another tensor while the entry lives (a cache keyed by
    data_ptr alone returned a previous grid's offsets when a freed buffer's address was reused -- found on the GPU)."""
    key = (offsets.data_ptr(), offsets.numel(), int(offsets._version))
    hit = _OFFSETS_HOST.get(key)
    if hit is None or hit[0] is not offsets:
        if len(_OFFSETS_HOST) > 64:
            _OFFSETS_HOST.clear()
        hit = _OFFSETS_HOST[key] = (offsets, np.ascontiguousarray(offsets.detach().cpu().numpy().astype(np.int32)))
    return hit[1]


def _all_half(what, **bufs):
    """The half instantiation reads every 16-bit buffer as at::Half (gridencoder.cu:468, 497): one of another dtype is refused
    before anything is launched, as the reference's data_ptr<scalar_t>() refuses it."""
    for name, t in bufs.items():
        if t is not None and (not torch.is_tensor(t) or t.dtype != torch.float16):
            raise RuntimeError(f"{what}: {name} must be float16 with a float16 table (got {getattr(t, 'dtype', type(t))})")


def _ck(rc, what):
    if rc != 0:
        # the reference raises RuntimeError (TORCH_CHECK / std::runtime_error)
        raise RuntimeError(f"{what}: {_capi.lib().gfpp_last_error().decode()}")


def _training_only(name):
    def f(*a, **k):
        raise NotImplementedError(f"{name} is a training-only op: keep the stock extension for training (SURVEY.md 2.2)")
    return f


def make_modules():
    L = _capi.lib()
    S = _capi.stream_ptr
    cf = ctypes.c_float

    rm = types.ModuleType("_raymarching_face")
    rm.near_far_from_aabb = lambda ro, rd, aabb, N, min_near, nears, fars: _ck(
        L.gfpp_near_far_from_aabb(_P(ro), _P(rd), _P(aabb), N, cf(min_near), _P(nears), _P(fars), S()), "near_far_from_aabb")
    rm.march_rays = lambda n_alive, n_step, alive, t, ro, rd, bound, dt_gamma, max_steps, C, H, grid, near, far, xyzs, dirs, deltas, noises: _ck(
        L.gfpp_march_rays(n_alive, n_step, _P(alive), _P(t), _P(ro), _P(rd), cf(bound), cf(dt_gamma), max_steps, C, H, _P(grid), _P(near),
                          _P(far), _P(xyzs), _P(dirs), _P(deltas), _P(noises), S()), "march_rays")
    rm.composite_rays = lambda n_alive, n_step, T_thresh, alive, t, sig, rgb, deltas, ws, depth, image: _ck(
        L.gfpp_composite_rays(n_alive, n_step, cf(T_thresh), _P(alive), _P(t), _P(sig), _P(rgb), _P(deltas), _P(ws), _P(depth), _P(image), S()),
        "composite_rays")
    # ---- training side (raymarching.h:8-17) ----
    scratch = {}

    def march_rays_train(ro, rd, grid, bound, dt_gamma, max_steps, N, C, H, M, nears, fars, xyzs, dirs, deltas, rays, counter, noises):
        need = L.gfpp_march_rays_train_scratch_bytes(N)
        key = ro.device.index
        if key not in scratch or scratch[key].numel() < need:
            scratch[key] = torch.empty(need, dtype=torch.uint8, device=ro.device)
        _ck(L.gfpp_march_rays_train(_P(ro), _P(rd), _P(grid), cf(bound), cf(dt_gamma), max_steps, N, C, H, M, _P(nears), _P(fars), _P(xyzs),
                                    _P(dirs), _P(deltas), _P(rays), _P(counter), _P(noises), _P(scratch[key]), scratch[key].numel(), S()),
            "march_rays_train")

    rm.march_rays_train = march_rays_train
    rm.march_rays_train_backward = lambda gx, gd, rays, deltas, N, M, gro, grd: _ck(
        L.gfpp_march_rays_train_backward(_P(gx), _P(gd), _P(rays), _P(deltas), N, M, _P(gro), _P(grd), S()), "march_rays_train_backward")
    rm.composite_rays_train_forward = lambda sig, rgb, amb, deltas, rays, M, N, T_thresh, ws, asum, depth, image: _ck(
        L.gfpp_composite_rays_train_forward(_P(sig), _P(rgb), _P(amb), _P(deltas), _P(rays), M, N, cf(T_thresh), _P(ws), _P(asum), _P(depth),
                                            _P(image), S()), "composite_rays_train_forward")
    rm.composite_rays_train_backward = lambda gws, gas, gimg, sig, rgb, amb, deltas, rays, ws, asum, image, M, N, T_thresh, gsig, grgb, gamb: _ck(
        L.gfpp_composite_rays_train_backward(_P(gws), _P(gas), _P(gimg), _P(sig), _P(rgb), _P(amb), _P(deltas), _P(rays), _P(ws), _P(asum),
                                             _P(image), M, N, cf(T_thresh), _P(gsig), _P(grgb), _P(gamb), S()), "composite_rays_train_backward")
    rm.packbits = lambda grid, N, thresh, bitfield: _ck(L.gfpp_packbits(_P(grid), N, cf(thresh), _P(bitfield), S()), "packbits")
    rm.morton3D = lambda coords, N, indices: _ck(L.gfpp_morton3D(_P(coords), N, _P(indices), S()), "morton3D")
    rm.morton3D_invert = lambda indices, N, coords: _ck(L.gfpp_morton3D_invert(_P(indices), N, _P(coords), S()), "morton3D_invert")
    rm.morton3D_dilation = lambda grid, C, H, out: _ck(L.gfpp_morton3D_dilation(_P(grid), C, H, _P(out), S()), "morton3D_dilation")
    rm.sph_from_ray = lambda ro, rd, radius, N, coords: _ck(L.gfpp_sph_from_ray(_P(ro), _P(rd), cf(radius), N, _P(coords), S()), "sph_from_ray")

    ge = types.ModuleType("_gridencoder")

    def grid_encode_forward(inputs, emb, offsets, outputs, B, D, C, Lv, S_, H, dy_dx, gridtype, align_corners, interp):
        if emb.dtype == torch.float16:   # autocast (grid.py:41-44): the reference's at::Half instantiation
            _all_half("grid_encode_forward", outputs=outputs, dy_dx=dy_dx)
            off = _offsets_host(offsets)
            _ck(L.gfpp_grid_encode_forward_half(_P(inputs, torch.float32), _P(emb, torch.float16), off.ctypes.data_as(ctypes.c_void_p),
                                                _P(outputs, torch.float16), B, D, C, Lv, cf(S_), H,
                                                None if dy_dx is None else _P(dy_dx, torch.float16), gridtype, int(align_corners), interp, S()),
                "grid_encode_forward")
            return
        if emb.dtype != torch.float32:
            raise RuntimeError(f"libgfpp grid tables are fp32 or fp16, not {emb.dtype}")
        off = _offsets_host(offsets)
        if dy_dx is not None:   # calc_grad_inputs (grid.py:49-52): the ambient grid's input comes out of the ambient net
            _ck(L.gfpp_grid_encode_forward_dydx(_P(inputs, torch.float32), _P(emb), off.ctypes.data_as(ctypes.c_void_p), _P(outputs, torch.float32),
                                                B, D, C, Lv, cf(S_), H, _P(dy_dx, torch.float32), gridtype, int(align_corners), interp, S()),
                "grid_encode_forward")
            return
        _ck(L.gfpp_grid_encode_forward(_P(inputs, torch.float32), _P(emb), off.ctypes.data_as(ctypes.c_void_p), _P(outputs, torch.float32), B, D, C, Lv, cf(S_), H, gridtype,
                                       int(align_corners), interp, S()), "grid_encode_forward")

    ge.grid_encode_forward = grid_encode_forward

    def grid_encode_backward(grad, inputs, emb, offsets, grad_emb, B, D, C, Lv, S_, H, dy_dx, grad_inputs, gridtype, align_corners, interp):
        if grad.dtype == torch.float16 or emb.dtype == torch.float16:   # the half instantiation: every 16-bit buffer must be half
            _all_half("grid_encode_backward", grad=grad, embeddings=emb, grad_embeddings=grad_emb, dy_dx=dy_dx, grad_inputs=grad_inputs)
            off = _offsets_host(offsets)
            _ck(L.gfpp_grid_encode_backward_half(_P(grad, torch.float16), _P(inputs, torch.float32), _P(emb, torch.float16),
                                                 off.ctypes.data_as(ctypes.c_void_p), _P(grad_emb, torch.float16), B, D, C, Lv, cf(S_), H,
                                                 None if dy_dx is None else _P(dy_dx, torch.float16),
                                                 None if grad_inputs is None else _P(grad_inputs, torch.float16), gridtype, int(align_corners),
                                                 interp, S()), "grid_encode_backward")
            return
        off = _offsets_host(offsets)
        _ck(L.gfpp_grid_encode_backward(_P(grad, torch.float32), _P(inputs, torch.float32), _P(emb, torch.float32), off.ctypes.data_as(ctypes.c_void_p),
                                        _P(grad_emb, torch.float32), B, D, C, Lv, cf(S_), H, None if dy_dx is None else _P(dy_dx, torch.float32),
                                        None if grad_inputs is None else _P(grad_inputs, torch.float32), gridtype, int(align_corners), interp, S()),
            "grid_encode_backward")

    def grad_total_variation(inputs, emb, grad, offsets, weight, B, D, C, Lv, S_, H, gridtype, align_corners):
        off = _offsets_host(offsets)
        _ck(L.gfpp_grad_total_variation(_P(inputs, torch.float32), _P(emb, torch.float32), _P(grad, torch.float32), off.ctypes.data_as(ctypes.c_void_p),
                                        cf(weight), B, D, C, Lv, cf(S_), H, gridtype, int(align_corners), S()), "grad_total_variation")

    ge.grid_encode_backward = grid_encode_backward
    ge.grad_total_variation = grad_total_variation

    sh = types.ModuleType("_shencoder")

    def sh_encode_forward(inp, out, B, D, C, dy_dx):
        if dy_dx is not None:
            raise NotImplementedError("sh_encode_forward with dy_dx is a training path")
        _ck(L.gfpp_sh_encode_forward(_P(inp), _P(out), B, D, C, S()), "sh_encode_forward")

    sh.sh_encode_forward = sh_encode_forward
    sh.sh_encode_backward = _training_only("sh_encode_backward")

    fr = types.ModuleType("_freqencoder")
    fr.freq_encode_forward = lambda inp, B, D, deg, C, out: _ck(L.gfpp_freq_encode_forward(_P(inp), B, D, deg, C, _P(out), S()), "freq_encode_forward")
    fr.freq_encode_backward = _training_only("freq_encode_backward")
    return {m.__name__: m for m in (rm, ge, sh, fr)}


def install():
    mods = make_modules()
    sys.modules.update(mods)
    return mods
