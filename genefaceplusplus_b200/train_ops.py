"""Training-side native ops on libgfpp (SURVEY.md 8(f) rank 4): the wrapper-level API of the reference's
modules/radnerfs/raymarching/raymarching.py:50-344 and encoders/gridencoder/grid.py:24-164 -- same function names, argument
meaning and autograd behaviour -- over csrc/train_kernels.cu through the C-ABI (include/gfpp.h section D).

    from genefaceplusplus_b200 import train_ops as raymarching
    xyzs, dirs, deltas, rays = raymarching.march_rays_train(rays_o, rays_d, bound, bitfield, C, H, nears, fars, counter, mean_count,
                                                            perturb, 128, force_all_rays, dt_gamma, max_steps)
    weights_sum, ambient_sum, depth, image = raymarching.composite_rays_train(sigmas, rgbs, ambient, deltas, rays, T_thresh)

`field` is RADNeRF.forward with its gradient (include/gfpp.h section G, csrc/field_train_kernel.cu, or with the model's
train_precision = "fp16" section J, csrc/field_train_tc_kernel.cu); RADNeRF.forward calls it.
`torso_field` is RADNeRFTorso.forward_torso with its gradient (section H); forward_torso calls it in training mode.
`torso_sr_field` is the same for RADNeRFTorsowithSR.forward_torso (section I).  Both run csrc/torso_train_kernel.cu, one source
instantiated for each field.

fp32 only (the reference casts with custom_fwd(cast_inputs=float32) as well); CUDA tensors only -- there is no CPU path.
Differences from the reference, both deliberate: march_rays_train lays the samples out in ray order (deterministic; the
reference's atomicAdd order changes from run to run, every consumer goes through `rays`), and nothing here calls
torch.cuda.empty_cache().
"""
import numpy as np
import torch
from torch.autograd import Function

import ctypes

from . import _capi, backend_shims

_mods = None


def _backend(name):
    global _mods
    if _mods is None:
        _mods = backend_shims.make_modules()
    return _mods[name]


def _cuda_f32(t):
    if not t.is_cuda:
        raise RuntimeError("libgfpp: expected a CUDA tensor (there is no CPU path)")
    return t.float().contiguous()


# ------------------------------------------------------------------------------------------------ update_extra_state helpers
def sph_from_ray(rays_o, rays_d, radius):
    """raymarching.py:50-78: [N,3] x2 -> [N,2] (theta, phi) in [-1,1] on the sphere of `radius`."""
    rays_o, rays_d = _cuda_f32(rays_o).view(-1, 3), _cuda_f32(rays_d).view(-1, 3)
    N = rays_o.shape[0]
    coords = torch.empty(N, 2, dtype=torch.float32, device=rays_o.device)
    _backend("_raymarching_face").sph_from_ray(rays_o, rays_d, radius, N, coords)
    return coords


def morton3D(coords):
    """raymarching.py:81-101: int32 [N,3] -> int32 [N]."""
    coords = coords.int().contiguous()
    indices = torch.empty(coords.shape[0], dtype=torch.int32, device=coords.device)
    _backend("_raymarching_face").morton3D(coords, coords.shape[0], indices)
    return indices


def morton3D_invert(indices):
    """raymarching.py:103-123: int32 [N] -> int32 [N,3]."""
    indices = indices.int().contiguous()
    coords = torch.empty(indices.shape[0], 3, dtype=torch.int32, device=indices.device)
    _backend("_raymarching_face").morton3D_invert(indices, indices.shape[0], coords)
    return coords


def packbits(grid, thresh, bitfield=None):
    """raymarching.py:126-152: float [C, H^3] -> uint8 [C*H^3/8], bit i of byte n = grid[8n+i] > thresh."""
    grid = _cuda_f32(grid)
    N = grid.shape[0] * grid.shape[1] // 8
    if bitfield is None:
        bitfield = torch.empty(N, dtype=torch.uint8, device=grid.device)
    _backend("_raymarching_face").packbits(grid, N, thresh, bitfield)
    return bitfield


def morton3D_dilation(grid):
    """raymarching.py:155-178: 6-neighbour max pooling of a Morton-ordered [C, H^3] grid."""
    grid = _cuda_f32(grid)
    C, H3 = grid.shape
    H = int(round(H3 ** (1.0 / 3.0)))
    out = torch.empty_like(grid)
    _backend("_raymarching_face").morton3D_dilation(grid, C, H, out)
    return out


# ------------------------------------------------------------------------------------------------ marching + compositing
def near_far_from_aabb(rays_o, rays_d, aabb, min_near=0.2):
    """raymarching.py:17-47: [N,3] x2 -> nears [N], fars [N] (both FLT_MAX on a miss)."""
    rays_o, rays_d = _cuda_f32(rays_o).view(-1, 3), _cuda_f32(rays_d).view(-1, 3)
    N = rays_o.shape[0]
    nears = torch.empty(N, dtype=torch.float32, device=rays_o.device)
    fars = torch.empty(N, dtype=torch.float32, device=rays_o.device)
    _backend("_raymarching_face").near_far_from_aabb(rays_o, rays_d, _cuda_f32(aabb), N, min_near, nears, fars)
    return nears, fars


class _march_rays_train(Function):
    """raymarching.py:184-273."""

    @staticmethod
    def forward(ctx, rays_o, rays_d, bound, density_bitfield, C, H, nears, fars, step_counter=None, mean_count=-1, perturb=False, align=-1,
                force_all_rays=False, dt_gamma=0, max_steps=1024):
        rays_o, rays_d = _cuda_f32(rays_o).view(-1, 3), _cuda_f32(rays_d).view(-1, 3)
        density_bitfield = density_bitfield.contiguous()
        dev = rays_o.device
        N = rays_o.shape[0]
        M = N * max_steps
        if not force_all_rays and mean_count > 0:
            if align > 0:
                mean_count += align - mean_count % align
            M = mean_count
        xyzs = torch.zeros(M, 3, dtype=torch.float32, device=dev)
        dirs = torch.zeros(M, 3, dtype=torch.float32, device=dev)
        deltas = torch.zeros(M, 2, dtype=torch.float32, device=dev)
        rays = torch.empty(N, 3, dtype=torch.int32, device=dev)
        if step_counter is None:
            step_counter = torch.zeros(2, dtype=torch.int32, device=dev)
        noises = torch.rand(N, dtype=torch.float32, device=dev) if perturb else torch.zeros(N, dtype=torch.float32, device=dev)
        _backend("_raymarching_face").march_rays_train(rays_o, rays_d, density_bitfield, bound, dt_gamma, max_steps, N, C, H, M, _cuda_f32(nears),
                                                       _cuda_f32(fars), xyzs, dirs, deltas, rays, step_counter, noises)
        if force_all_rays or mean_count <= 0:
            m = int(step_counter[0].item())
            if align > 0:
                m += align - m % align
            xyzs, dirs, deltas = xyzs[:m], dirs[:m], deltas[:m]
        ctx.save_for_backward(rays, deltas)
        ctx.mark_non_differentiable(rays)
        return xyzs, dirs, deltas, rays

    @staticmethod
    def backward(ctx, grad_xyzs, grad_dirs, grad_deltas, grad_rays):
        rays, deltas = ctx.saved_tensors
        N, M = rays.shape[0], grad_xyzs.shape[0]
        grad_rays_o = torch.zeros(N, 3, device=rays.device)
        grad_rays_d = torch.zeros(N, 3, device=rays.device)
        _backend("_raymarching_face").march_rays_train_backward(_cuda_f32(grad_xyzs), _cuda_f32(grad_dirs), rays, deltas.contiguous(), N, M,
                                                                grad_rays_o, grad_rays_d)
        return (grad_rays_o, grad_rays_d) + (None,) * 13


march_rays_train = _march_rays_train.apply


class _composite_rays_train(Function):
    """raymarching.py:276-341 (grad_depth is not propagated there either)."""

    @staticmethod
    def forward(ctx, sigmas, rgbs, ambient, deltas, rays, T_thresh=1e-4):
        sigmas, rgbs, ambient, deltas = _cuda_f32(sigmas), _cuda_f32(rgbs), _cuda_f32(ambient), _cuda_f32(deltas)
        M, N = sigmas.shape[0], rays.shape[0]
        dev = sigmas.device
        weights_sum = torch.empty(N, dtype=torch.float32, device=dev)
        ambient_sum = torch.empty(N, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        image = torch.empty(N, 3, dtype=torch.float32, device=dev)
        _backend("_raymarching_face").composite_rays_train_forward(sigmas, rgbs, ambient, deltas, rays, M, N, T_thresh, weights_sum, ambient_sum, depth, image)
        ctx.save_for_backward(sigmas, rgbs, ambient, deltas, rays, weights_sum, ambient_sum, image)
        ctx.dims = [M, N, T_thresh]
        return weights_sum, ambient_sum, depth, image

    @staticmethod
    def backward(ctx, grad_weights_sum, grad_ambient_sum, grad_depth, grad_image):
        sigmas, rgbs, ambient, deltas, rays, weights_sum, ambient_sum, image = ctx.saved_tensors
        M, N, T_thresh = ctx.dims
        grad_sigmas, grad_rgbs, grad_ambient = torch.zeros_like(sigmas), torch.zeros_like(rgbs), torch.zeros_like(ambient)
        _backend("_raymarching_face").composite_rays_train_backward(_cuda_f32(grad_weights_sum), _cuda_f32(grad_ambient_sum), _cuda_f32(grad_image), sigmas, rgbs,
                                                                    ambient, deltas, rays, weights_sum, ambient_sum, image, M, N, T_thresh, grad_sigmas,
                                                                    grad_rgbs, grad_ambient)
        return grad_sigmas, grad_rgbs, grad_ambient, None, None, None


composite_rays_train = _composite_rays_train.apply


# ------------------------------------------------------------------------------------------------ grid encoder with gradients
class _grid_encode(Function):
    """grid.py:24-88: inputs [B,D] in [0,1], embeddings [sum,C] -> [B, L*C]; gradients w.r.t. the table (vector reductions) and,
    with calc_grad_inputs, w.r.t. the inputs (through dy_dx)."""

    @staticmethod
    def forward(ctx, inputs, embeddings, offsets, per_level_scale, base_resolution, calc_grad_inputs=False, gridtype=0, align_corners=False,
                interpolation=0):
        inputs, embeddings = _cuda_f32(inputs), _cuda_f32(embeddings)
        B, D = inputs.shape
        L, C = offsets.shape[0] - 1, embeddings.shape[1]
        S = float(np.log2(per_level_scale))
        outputs = torch.empty(L, B, C, device=inputs.device, dtype=torch.float32)
        dy_dx = torch.empty(B, L * D * C, device=inputs.device, dtype=torch.float32) if calc_grad_inputs else None
        _backend("_gridencoder").grid_encode_forward(inputs, embeddings, offsets, outputs, B, D, C, L, S, base_resolution, dy_dx, gridtype, align_corners,
                                                     interpolation)
        ctx.save_for_backward(inputs, embeddings, offsets, dy_dx)
        ctx.dims = [B, D, C, L, S, base_resolution, gridtype, interpolation, align_corners]
        return outputs.permute(1, 0, 2).reshape(B, L * C)

    @staticmethod
    def backward(ctx, grad):
        inputs, embeddings, offsets, dy_dx = ctx.saved_tensors
        B, D, C, L, S, H, gridtype, interpolation, align_corners = ctx.dims
        grad = _cuda_f32(grad).view(B, L, C).permute(1, 0, 2).contiguous()
        grad_embeddings = torch.zeros_like(embeddings)
        grad_inputs = torch.zeros_like(inputs) if dy_dx is not None else None
        _backend("_gridencoder").grid_encode_backward(grad, inputs, embeddings, offsets, grad_embeddings, B, D, C, L, S, H, dy_dx, grad_inputs, gridtype,
                                                      align_corners, interpolation)
        return grad_inputs, grad_embeddings, None, None, None, None, None, None, None


grid_encode = _grid_encode.apply


@torch.no_grad()
def grad_total_variation(embeddings, offsets, per_level_scale, base_resolution, input_dim, weight=1e-7, inputs=None, bound=1, B=1000000, gridtype=0,
                         align_corners=False):
    """GridEncoder.grad_total_variation (grid.py:166-185): adds the TV gradient of the cells `inputs` fall into (random points when
    None) to embeddings.grad, which must exist."""
    if embeddings.grad is None:
        raise ValueError("grad is None, should be called after loss.backward() and before optimizer.step()!")
    D, C, L = input_dim, embeddings.shape[1], offsets.shape[0] - 1
    if inputs is None:
        inputs = torch.rand(B, D, device=embeddings.device)
    else:
        inputs = (inputs + bound) / (2 * bound)
        inputs = inputs.view(-1, D)
        B = inputs.shape[0]
    _backend("_gridencoder").grad_total_variation(_cuda_f32(inputs), _cuda_f32(embeddings), embeddings.grad, offsets, weight, B, D, C, L,
                                                  float(np.log2(per_level_scale)), base_resolution, gridtype, align_corners)


# ------------------------------------------------------------------------------------------------ shared by the training fields
def _workspace(model, attr, bytes_fn, M, what):
    """The device workspace of `bytes_fn(M)` bytes, cached on the model as `attr` and regrown when too small."""
    need = bytes_fn(M)
    if need == 0:
        raise _capi.GfppError(f"{what} does not support {M} points per call")
    dev = model.density_bitfield.device
    ws = model.__dict__.get(attr)
    if ws is None or ws.numel() < need or ws.device != dev:
        ws = model.__dict__[attr] = torch.empty(need, dtype=torch.uint8, device=dev)
    return ws


def _host_offsets(gp):
    """The grid's level offsets as a host int32 array, copied from the device once per offsets buffer (they never change in training)."""
    key = (gp.offsets.data_ptr(), gp.offsets._version)
    cached = gp.__dict__.get("_host_offsets")
    if cached is None or cached[0] != key:
        cached = gp.__dict__["_host_offsets"] = (key, np.ascontiguousarray(gp.offsets.detach().cpu().numpy().astype(np.int32)))
    return cached[1]


def _fill_grid(g, gp, emb, keep):
    """Fills the gfpp_grid_desc `g` for the _GridParams `gp` with table `emb` and the cached host offsets."""
    lay = gp.layout
    off = _host_offsets(gp)
    keep += [emb, off]
    g.embeddings, g.offsets_host = emb.data_ptr(), off.ctypes.data
    g.input_dim, g.num_levels, g.base_resolution = lay.input_dim, lay.num_levels, lay.base_resolution
    g.log2_per_level_scale, g.gridtype, g.interp, g.align_corners = float(lay.S), lay.gridtype_id, lay.interp_id, int(lay.align_corners)


def _backward_buffers(M, dev, upstream, shapes, targets, code, tables):
    """The common start of the fields' backward: the upstream gradients as contiguous fp32 of `shapes` (zeros where autograd passes
    None), and fp32 gradient buffers shaped like `targets` and like `code` (None without a code).  The kernels write every element
    of these buffers except the grid tables' (indices `tables` of `targets`), which they accumulate into; with M = 0 no kernel
    runs, so all of them are zeros."""
    up = [torch.zeros(s, device=dev) if g is None else _cuda_f32(g).reshape(s) for g, s in zip(upstream, shapes)]

    def buf(t, accumulated=False):
        return (torch.zeros if M == 0 or accumulated else torch.empty)(t.shape, dtype=torch.float32, device=dev)

    return up, [buf(t, i in tables) for i, t in enumerate(targets)], None if code is None else buf(code)


# ------------------------------------------------------------------------------------------------ the head field
# model.train_precision -> (workspace attribute, workspace-size, forward and backward entry points); the two sets take the same arguments
_FIELD_ENTRY = {"fp32": ("_field_ws", "gfpp_field_backward_workspace_bytes", "gfpp_field_forward", "gfpp_field_backward"),
                "fp16": ("_field_tc_ws", "gfpp_field_tc_workspace_bytes", "gfpp_field_tc_forward", "gfpp_field_tc_backward")}


def _field_workspace(model, entry, M):
    return _workspace(model, entry[0], getattr(_capi.lib(), entry[1]), M, "the training field")


def _field_desc(model, code, keep):
    """The gfpp_model_desc fields section (G) reads -- grids, weights, code, cond_dim, bound, precision -- with no device-to-host copy."""
    d = _capi.ModelDesc()
    for name, gp in (("position_grid", model.position_embedder), ("ambient_grid", model.ambient_embedder)):
        _fill_grid(getattr(d, name), gp, _cuda_f32(gp.embeddings.detach()), keep)
    ws = [_cuda_f32(w.weight.detach()) for w in list(model.ambient_net.net) + list(model.sigma_net.net) + list(model.color_net.net)]
    keep += ws
    for i in range(3):
        d.ambient_w[i], d.sigma_w[i] = ws[i].data_ptr(), ws[3 + i].data_ptr()
    d.color_w[0], d.color_w[1] = ws[6].data_ptr(), ws[7].data_ptr()
    d.individual_code = code.data_ptr() if code is not None else None
    d.cond_dim, d.ind_dim = model.cond_out_dim, model.individual_embedding_dim
    d.bound = float(model.bound)
    d.mlp_precision = 0
    return d


class _field(Function):
    """RADNeRF.forward (radnerf.py:108-141) over gfpp_field_forward / gfpp_field_backward: (xyzs [M,3], dirs [M,3], cond_feat [64] or
    [1,64], code [ind_dim] or None) -> (sigma [M], color [M,3], ambient_pos [M,A]).  `params` are the eight MLP weights and the two grid
    tables of `model`, passed so that autograd routes their gradients; the kernels read them in place.  No gradient reaches xyzs or
    dirs (the caller rejects inputs that require one).  model.train_precision picks the entry points (_FIELD_ENTRY) at the forward;
    the backward uses the same ones."""

    @staticmethod
    def forward(ctx, model, xyzs, dirs, cond_feat, code, *params):
        if model.train_precision not in _FIELD_ENTRY:
            raise ValueError(f'train_precision must be "fp32" or "fp16", got {model.train_precision!r}')
        entry = ctx.entry = _FIELD_ENTRY[model.train_precision]
        x, dr = _cuda_f32(xyzs).view(-1, 3), _cuda_f32(dirs).view(-1, 3)
        if cond_feat.numel() != model.cond_out_dim:
            raise ValueError(f"cond_feat must hold one conditioning vector of {model.cond_out_dim} values, got shape {tuple(cond_feat.shape)}")
        if (code is None) != (model.individual_embedding_dim == 0) or (code is not None and code.numel() != model.individual_embedding_dim):
            raise ValueError(f"individual_code must hold {model.individual_embedding_dim} values (None iff the model has no codes)")
        c = _cuda_f32(cond_feat).reshape(-1)
        cd = _cuda_f32(code).reshape(-1) if code is not None else None
        M, A, dev = x.shape[0], model.ambient_coord_dim, x.device
        sigma = torch.empty(M, dtype=torch.float32, device=dev)
        color = torch.empty(M, 3, dtype=torch.float32, device=dev)
        amb = torch.empty(M, A, dtype=torch.float32, device=dev)
        keep = []
        d = _field_desc(model, cd, keep)
        ws = _field_workspace(model, entry, 0)
        with torch.cuda.device(dev):
            _capi.check(getattr(_capi.lib(), entry[2])(ctypes.byref(d), x.data_ptr(), dr.data_ptr(), M, c.data_ptr(), sigma.data_ptr(), color.data_ptr(),
                                                       amb.data_ptr(), ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), entry[2])
        ctx.model = model
        ctx.shapes = (cond_feat.shape, None if code is None else code.shape)
        ctx.save_for_backward(x, dr, c, cd if cd is not None else torch.empty(0, device=dev), *params)
        return sigma, color, amb

    @staticmethod
    def backward(ctx, g_sigma, g_color, g_amb):
        x, dr, c, cd, *params = ctx.saved_tensors
        model = ctx.model
        cond_shape, code_shape = ctx.shapes
        M, dev = x.shape[0], x.device
        (g_sigma, g_color, g_amb), grads, g_code = _backward_buffers(M, dev, (g_sigma, g_color, g_amb), ((M,), (M, 3), (M, model.ambient_coord_dim)),
                                                                     [*params, c], None if code_shape is None else cd, tables=(8, 9))
        grad_w, g_pos, g_tab, g_cond = grads[:8], grads[8], grads[9], grads[10]
        keep = []
        d = _field_desc(model, cd if code_shape is not None else None, keep)
        ws = _field_workspace(model, ctx.entry, M)
        ptrs = (ctypes.c_void_p * 8)(*[g.data_ptr() for g in grad_w])
        with torch.cuda.device(dev):
            _capi.check(getattr(_capi.lib(), ctx.entry[3])(ctypes.byref(d), x.data_ptr(), dr.data_ptr(), M, c.data_ptr(), g_sigma.data_ptr(),
                                                           g_color.data_ptr(), g_amb.data_ptr(), ctypes.byref(ptrs), g_cond.data_ptr(),
                                                           None if g_code is None else g_code.data_ptr(), g_pos.data_ptr(), g_tab.data_ptr(),
                                                           ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), ctx.entry[3])
        grads = [g.to(p.dtype) for g, p in zip(grads, params)]
        return (None, None, None, g_cond.view(cond_shape), None if g_code is None else g_code.view(code_shape), *grads)


field = _field.apply


# ------------------------------------------------------------------------------------------------ the torso field
def _torso_field_workspace(model, M):
    return _workspace(model, "_torso_field_ws", _capi.lib().gfpp_torso_field_workspace_bytes, M, "the torso training field")


def _torso_field_desc(model, keep):
    """The gfpp_model_desc fields section (H) reads -- torso grid, the six torso weights, torso_code_dim, torso_shrink -- with no
    device-to-host copy."""
    d = _capi.ModelDesc()
    _fill_grid(d.torso_grid, model.torso_embedder, _cuda_f32(model.torso_embedder.embeddings.detach()), keep)
    ws = [_cuda_f32(w.weight.detach()) for w in list(model.torso_deform_net.net) + list(model.torso_canonicial_net.net)]
    keep += ws
    for i in range(3):
        d.torso_deform_w[i], d.torso_canon_w[i] = ws[i].data_ptr(), ws[3 + i].data_ptr()
    d.torso_code_dim = model.torso_individual_embedding_dim
    d.torso_shrink = float(model.torso_shrink)
    return d


class _torso_field(Function):
    """RADNeRFTorso.forward_torso (radnerf_torso.py:51-84) over gfpp_torso_field_forward / gfpp_torso_field_backward: (x [M,2] in
    [-1,1], pose6 [6] or [1,6], code [torso_code_dim] or [1,torso_code_dim] or None) -> (alpha [M,1], color [M,3], dx [M,2]).  `params`
    are the six torso MLP weights and the torso grid table of `model`, passed so that autograd routes their gradients; the kernels
    read them in place.  `code` may be a view such as torso_individual_codes[index]: autograd then routes its gradient to that row
    only.  No gradient reaches x or the pose (the caller rejects inputs that require one)."""

    @staticmethod
    def forward(ctx, model, x, pose6, code, *params):
        xy = _cuda_f32(x).view(-1, 2)
        p6 = _cuda_f32(pose6).reshape(-1)
        if p6.numel() != 6:
            raise ValueError(f"forward_torso takes one pose [1,6] (convert_poses), got shape {tuple(pose6.shape)}")
        cdim = model.torso_individual_embedding_dim
        if (code is None) != (cdim == 0) or (code is not None and code.numel() != cdim):
            raise ValueError(f"c must hold {cdim} values (None iff the model has no torso_individual_codes)")
        cd = _cuda_f32(code).reshape(-1) if code is not None else None
        M, dev = xy.shape[0], xy.device
        alpha = torch.empty(M, 1, dtype=torch.float32, device=dev)
        color = torch.empty(M, 3, dtype=torch.float32, device=dev)
        dx = torch.empty(M, 2, dtype=torch.float32, device=dev)
        keep = []
        d = _torso_field_desc(model, keep)
        ws = _torso_field_workspace(model, 0)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_field_forward(ctypes.byref(d), xy.data_ptr(), M, p6.data_ptr(), None if cd is None else cd.data_ptr(),
                                                             alpha.data_ptr(), color.data_ptr(), dx.data_ptr(), ws.data_ptr(), ws.numel(),
                                                             _capi.stream_ptr(dev)), "gfpp_torso_field_forward")
        ctx.model = model
        ctx.code_shape = None if code is None else code.shape
        ctx.save_for_backward(xy, p6, cd if cd is not None else torch.empty(0, device=dev), *params)
        return alpha, color, dx

    @staticmethod
    def backward(ctx, g_alpha, g_color, g_dx):
        xy, p6, cd, *params = ctx.saved_tensors
        model, code_shape = ctx.model, ctx.code_shape
        M, dev = xy.shape[0], xy.device
        (g_alpha, g_color, g_dx), grads, g_code = _backward_buffers(M, dev, (g_alpha, g_color, g_dx), ((M,), (M, 3), (M, 2)), params,
                                                                    None if code_shape is None else cd, tables=(6,))
        keep = []
        d = _torso_field_desc(model, keep)
        ws = _torso_field_workspace(model, M)
        p_def = (ctypes.c_void_p * 3)(*[g.data_ptr() for g in grads[:3]])
        p_can = (ctypes.c_void_p * 3)(*[g.data_ptr() for g in grads[3:6]])
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_field_backward(ctypes.byref(d), xy.data_ptr(), M, p6.data_ptr(),
                                                              None if code_shape is None else cd.data_ptr(), g_alpha.data_ptr(),
                                                              g_color.data_ptr(), g_dx.data_ptr(), ctypes.byref(p_def), ctypes.byref(p_can),
                                                              None if g_code is None else g_code.data_ptr(), grads[6].data_ptr(), ws.data_ptr(),
                                                              ws.numel(), _capi.stream_ptr(dev)), "gfpp_torso_field_backward")
        grads = [g.to(p.dtype) for g, p in zip(grads, params)]
        return (None, None, None, None if g_code is None else g_code.view(code_shape), *grads)


torso_field = _torso_field.apply


# ------------------------------------------------------------------------------------------------ the torso-SR field
def _torso_sr_field_workspace(model, M):
    return _workspace(model, "_torso_sr_field_ws", _capi.lib().gfpp_torso_sr_field_workspace_bytes, M, "the torso-SR training field")


def torso_sr_params(model):
    """The parameters of RADNeRFTorsowithSR's torso field in the order torso_sr_field takes them: the six torso MLP weights, the torso
    grid table and, with torso_head_aware, the three weights then the three biases of head_color_weights_encoder."""
    p = ([model.torso_deform_net.net[i].weight for i in range(3)] + [model.torso_canonicial_net.net[i].weight for i in range(3)] +
         [model.torso_embedder.embeddings])
    if model.torso_head_aware:
        lins = [model.head_color_weights_encoder[i] for i in (0, 2, 4)]
        p += [lin.weight for lin in lins] + [lin.bias for lin in lins]
    return p


def _torso_sr_field_desc(model, params, keep):
    """The gfpp_torso_sr_desc fields section (I) reads -- torso grid, the six torso weights, torso_code_dim, head_aware and the
    encoder, torso_shrink -- from `params` (torso_sr_params order), with no device-to-host copy."""
    d = _capi.TorsoSrDesc()
    ws = [_cuda_f32(p.detach()) for p in params]
    keep += ws
    _fill_grid(d.torso_grid, model.torso_embedder, ws[6], keep)
    for i in range(3):
        d.torso_deform_w[i], d.torso_canon_w[i] = ws[i].data_ptr(), ws[3 + i].data_ptr()
    d.torso_code_dim = model.torso_individual_embedding_dim
    d.head_aware = int(model.torso_head_aware)
    if model.torso_head_aware:
        for i in range(3):
            d.ha_w[i], d.ha_b[i] = ws[7 + i].data_ptr(), ws[10 + i].data_ptr()
    d.torso_shrink = float(model.torso_shrink)
    return d


class _torso_sr_field(Function):
    """RADNeRFTorsowithSR.forward_torso (radnerf_torso_sr.py:75-114) over gfpp_torso_sr_field_forward / gfpp_torso_sr_field_backward:
    (x [M,2] in [-1,1], lm68 (136 values), code [torso_code_dim] or [1,torso_code_dim] or None, image [M,3] and weights_sum [M,1] /
    [M] or both None) -> (alpha [M,1], color [M,3], dx [M,2]).  image and weights_sum are read only with torso_head_aware (None:
    zeros, the reference's image=None path).  `params` are the model's torso_sr_params, passed so that autograd routes their
    gradients; the kernels read them in place.  `code` may be a view such as torso_individual_codes[index]: autograd then routes
    its gradient to that row only.  No gradient reaches x, lm68, image or weights_sum (the caller rejects inputs that require one)."""

    @staticmethod
    def forward(ctx, model, x, lm68, code, image, weights_sum, *params):
        xy = _cuda_f32(x).view(-1, 2)
        lm = _cuda_f32(lm68).reshape(-1)
        if lm.numel() != 136:
            raise ValueError(f"lm68 must hold the 68 2-D landmarks of one frame (136 values), got shape {tuple(lm68.shape)}")
        cdim = model.torso_individual_embedding_dim
        if (code is None) != (cdim == 0) or (code is not None and code.numel() != cdim):
            raise ValueError(f"c must hold {cdim} values (None iff the model has no torso_individual_codes)")
        M, dev = xy.shape[0], xy.device
        if not model.torso_head_aware:
            image = weights_sum = None                      # the reference ignores them without torso_head_aware
        if (image is None) != (weights_sum is None):
            raise ValueError("image and weights_sum must both be given or both be None")
        img = ws_ = None
        if image is not None:
            img, ws_ = _cuda_f32(image).reshape(-1, 3), _cuda_f32(weights_sum).reshape(-1)
            if img.shape[0] != M or ws_.numel() != M:
                raise ValueError(f"image must be [{M},3] and weights_sum [{M},1], got {tuple(image.shape)} and {tuple(weights_sum.shape)}")
        cd = _cuda_f32(code).reshape(-1) if code is not None else None
        alpha = torch.empty(M, 1, dtype=torch.float32, device=dev)
        color = torch.empty(M, 3, dtype=torch.float32, device=dev)
        dx = torch.empty(M, 2, dtype=torch.float32, device=dev)
        keep = []
        d = _torso_sr_field_desc(model, params, keep)
        ws = _torso_sr_field_workspace(model, 0)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_sr_field_forward(ctypes.byref(d), xy.data_ptr(), M, lm.data_ptr(), None if cd is None else cd.data_ptr(),
                                                                None if img is None else img.data_ptr(), None if ws_ is None else ws_.data_ptr(),
                                                                alpha.data_ptr(), color.data_ptr(), dx.data_ptr(), ws.data_ptr(), ws.numel(),
                                                                _capi.stream_ptr(dev)), "gfpp_torso_sr_field_forward")
        ctx.model = model
        ctx.code_shape = None if code is None else code.shape
        ctx.has_image = img is not None
        empty = torch.empty(0, device=dev)
        ctx.save_for_backward(xy, lm, cd if cd is not None else empty, img if img is not None else empty, ws_ if ws_ is not None else empty, *params)
        return alpha, color, dx

    @staticmethod
    def backward(ctx, g_alpha, g_color, g_dx):
        xy, lm, cd, img, ws_, *params = ctx.saved_tensors
        model, code_shape = ctx.model, ctx.code_shape
        M, dev = xy.shape[0], xy.device
        (g_alpha, g_color, g_dx), grads, g_code = _backward_buffers(M, dev, (g_alpha, g_color, g_dx), ((M,), (M, 3), (M, 2)), params,
                                                                    None if code_shape is None else cd, tables=(6,))
        keep = []
        d = _torso_sr_field_desc(model, params, keep)
        ws = _torso_sr_field_workspace(model, M)
        P3 = ctypes.c_void_p * 3
        p_def, p_can = P3(*[g.data_ptr() for g in grads[:3]]), P3(*[g.data_ptr() for g in grads[3:6]])
        p_haw = P3(*[g.data_ptr() for g in grads[7:10]]) if len(grads) > 7 else None
        p_hab = P3(*[g.data_ptr() for g in grads[10:13]]) if len(grads) > 7 else None
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_sr_field_backward(
                ctypes.byref(d), xy.data_ptr(), M, lm.data_ptr(), None if code_shape is None else cd.data_ptr(),
                img.data_ptr() if ctx.has_image else None, ws_.data_ptr() if ctx.has_image else None, g_alpha.data_ptr(), g_color.data_ptr(),
                g_dx.data_ptr(), ctypes.byref(p_def), ctypes.byref(p_can), None if p_haw is None else ctypes.byref(p_haw),
                None if p_hab is None else ctypes.byref(p_hab), None if g_code is None else g_code.data_ptr(), grads[6].data_ptr(),
                ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_torso_sr_field_backward")
        grads = [g.to(p.dtype) for g, p in zip(grads, params)]
        return (None, None, None, None if g_code is None else g_code.view(code_shape), None, None, *grads)


torso_sr_field = _torso_sr_field.apply


# ------------------------------------------------------------------------------------------------ the torso pass of the torso steps
def _composite_forward(slot, M, alpha, color, img, ws, bg, bg_mode):
    """gfpp_torso_composite_forward: (torso_alpha_map [N,1], torso_rgb_map [N,3], rgb_map [N,3]); alpha / color None iff M == 0."""
    N, dev = slot.shape[0], slot.device
    ta = torch.empty(N, 1, dtype=torch.float32, device=dev)
    trgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
    rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
    _capi.check(_capi.lib().gfpp_torso_composite_forward(slot.data_ptr(), N, M, None if alpha is None else alpha.data_ptr(),
                                                         None if color is None else color.data_ptr(), img.data_ptr(), ws.data_ptr(),
                                                         None if bg is None else bg.data_ptr(), bg_mode, ta.data_ptr(), trgb.data_ptr(),
                                                         rgb.data_ptr(), _capi.stream_ptr(dev)), "gfpp_torso_composite_forward")
    return ta, trgb, rgb


class _torso_composite(Function):
    """The three-way composite of the torso steps (radnerf_torso.py:172-193) over gfpp_torso_composite_forward / _backward: the field's
    alpha [M,1] and color [M,3] at the masked pixels (slot [N], idx [M] of gfpp_torso_mask), the head image [N,3], weights_sum [N] and
    the background (bg_mode 0: None, 1: bg [3], 2: bg [N,3]) -> (torso_alpha_map [N,1], torso_rgb_map [N,3], rgb_map [N,3]).  Gradients
    reach alpha and color only (the caller rejects other inputs that require one)."""

    @staticmethod
    def forward(ctx, slot, idx, img, ws, bg, bg_mode, alpha, color):
        a, c = alpha.contiguous().reshape(-1), color.contiguous().reshape(-1, 3)
        with torch.cuda.device(slot.device):
            out = _composite_forward(slot, a.shape[0], a, c, img, ws, bg, bg_mode)
        ctx.bg_mode = bg_mode
        ctx.save_for_backward(idx, img, ws, bg if bg is not None else torch.empty(0, device=slot.device), a, c)
        return out

    @staticmethod
    def backward(ctx, g_ta, g_trgb, g_rgb):
        idx, img, ws, bg, a, c = ctx.saved_tensors
        N, M, dev = ws.shape[0], a.shape[0], a.device
        grad_alpha = torch.empty(M, 1, dtype=torch.float32, device=dev)
        grad_color = torch.empty(M, 3, dtype=torch.float32, device=dev)
        ups = [None if g is None else _cuda_f32(g) for g in (g_ta, g_trgb, g_rgb)]
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_composite_backward(
                idx.data_ptr(), N, M, a.data_ptr(), c.data_ptr(), img.data_ptr(), ws.data_ptr(), bg.data_ptr() if ctx.bg_mode else None,
                ctx.bg_mode, *[None if g is None else g.data_ptr() for g in ups], grad_alpha.data_ptr(), grad_color.data_ptr(),
                _capi.stream_ptr(dev)), "gfpp_torso_composite_backward")
        return None, None, None, None, None, None, grad_alpha, grad_color


def _count_host(model):
    """A pinned host int32 that receives M (kept on the model across calls)."""
    h = model.__dict__.get("_torso_pass_count")
    if h is None:
        h = model.__dict__["_torso_pass_count"] = torch.empty(1, dtype=torch.int32, pin_memory=True)
    return h


def torso_pass(model, image, weights_sum, bg_coords, bg_color, field, head_aware):
    """The torso part of the torso training steps (radnerf_torso.py:165-193, radnerf_torso_sr.py:196-221) on gfpp.h section M:
    mask + compaction (gfpp_torso_mask), one device-to-host read of M, field(xy [M,2], image [M,3], weights_sum [M]) -> (alpha [M,1],
    color [M,3], deform [M,2]) on the masked pixels (the autograd Function of section H or I; image and weights_sum gathered iff
    head_aware, None otherwise), then the composite (_torso_composite).  Returns the composed recipe's dict: torso_alpha_map [N,1],
    torso_rgb_map [N,3], rgb_map [N,3] (clamped), weights_sum [N] and, iff M > 0, deform [M,2].  With M == 0 no field runs and no
    output requires grad (the reference's `if mask.any()`).  Sets model.last_launch_count.  Shapes are checked (ValueError) before
    anything reaches the device; the caller has checked that nothing but the field's parameters requires grad."""
    N = bg_coords.numel() // 2
    if N == 0 or bg_coords.numel() != 2 * N or bg_coords.shape[-1] != 2:
        raise ValueError(f"bg_coords must be [...,2] with at least one pixel, got shape {tuple(bg_coords.shape)}")
    if image.numel() != 3 * N or weights_sum.numel() != N:
        raise ValueError(f"image must hold {N}x3 values and weights_sum {N} (one per pixel of bg_coords), got shapes "
                         f"{tuple(image.shape)} and {tuple(weights_sum.shape)}")
    bg_mode = 0
    if bg_color is not None:
        bg_mode = 1 if bg_color.numel() == 3 else 2 if bg_color.numel() == 3 * N else -1
        if bg_mode < 0:
            raise ValueError(f"bg_color must be None, one colour (3 values) or one per pixel ({N}x3), got shape {tuple(bg_color.shape)}")
    L = _capi.lib()
    dev = model.density_bitfield.device
    f32 = torch.float32
    grid = model.density_grid_torso
    if grid.dtype != f32 or not grid.is_contiguous() or grid.device != dev:
        raise ValueError("density_grid_torso must be a contiguous fp32 buffer on the model's device")
    xy = bg_coords.detach().to(dev, f32).reshape(N, 2).contiguous()
    img = image.detach().to(dev, f32).reshape(N, 3).contiguous()
    ws = weights_sum.detach().to(dev, f32).reshape(N).contiguous()
    bg = None if bg_color is None else bg_color.detach().to(dev, f32).reshape(-1).contiguous()
    i32 = torch.int32
    idx, slot, count = torch.empty(N, dtype=i32, device=dev), torch.empty(N, dtype=i32, device=dev), torch.empty(1, dtype=i32, device=dev)
    xy_m = torch.empty(N, 2, dtype=f32, device=dev)
    img_m = torch.empty(N, 3, dtype=f32, device=dev) if head_aware else None
    ws_m = torch.empty(N, dtype=f32, device=dev) if head_aware else None
    work = _workspace(model, "_torso_pass_ws", L.gfpp_torso_pass_workspace_bytes, N, "the torso pass")
    # the mask threshold as PyTorch compares it: the Python float min() rounded to float32 (the c_float argument)
    thr = float(min(model.density_thresh_torso, model.mean_density_torso))
    host = _count_host(model)
    with torch.cuda.device(dev):
        _capi.check(L.gfpp_torso_mask(grid.data_ptr(), model.grid_size, thr, xy.data_ptr(), N, img.data_ptr() if head_aware else None,
                                      ws.data_ptr() if head_aware else None, idx.data_ptr(), slot.data_ptr(), xy_m.data_ptr(),
                                      None if img_m is None else img_m.data_ptr(), None if ws_m is None else ws_m.data_ptr(), count.data_ptr(),
                                      work.data_ptr(), work.numel(), _capi.stream_ptr(dev)), "gfpp_torso_mask")
        launches = int(L.gfpp_last_launch_count())
        host.copy_(count, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()               # the one host sync of the pass: M sizes the field's launch and its outputs
        M = int(host[0])
        if M == 0:
            ta, trgb, rgb = _composite_forward(slot, 0, None, None, img, ws, bg, bg_mode)
            model.last_launch_count = launches + 1
            return {"torso_alpha_map": ta, "torso_rgb_map": trgb, "rgb_map": rgb, "weights_sum": ws}
    alpha, color, deform = field(xy_m[:M], None if img_m is None else img_m[:M], None if ws_m is None else ws_m[:M])
    launches += int(L.gfpp_last_launch_count())
    ta, trgb, rgb = _torso_composite.apply(slot, idx[:M], img, ws, bg, bg_mode, alpha, color)
    model.last_launch_count = launches + 1
    return {"torso_alpha_map": ta, "torso_rgb_map": trgb, "rgb_map": rgb, "weights_sum": ws, "deform": deform}
