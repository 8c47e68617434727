"""Training-side native ops on libgfpp (SURVEY.md 8(f) rank 4): the wrapper-level API of the reference's
modules/radnerfs/raymarching/raymarching.py:50-344 and encoders/gridencoder/grid.py:24-164 -- same function names, argument
meaning and autograd behaviour -- over csrc/train_kernels.cu through the C-ABI (include/gfpp.h section D).

    from genefaceplusplus_b200 import train_ops as raymarching
    xyzs, dirs, deltas, rays = raymarching.march_rays_train(rays_o, rays_d, bound, bitfield, C, H, nears, fars, counter, mean_count,
                                                            perturb, 128, force_all_rays, dt_gamma, max_steps)
    weights_sum, ambient_sum, depth, image = raymarching.composite_rays_train(sigmas, rgbs, ambient, deltas, rays, T_thresh)

`field` is RADNeRF.forward with its gradient (include/gfpp.h section G, csrc/field_train_kernel.cu); RADNeRF.forward calls it.
`torso_field` is RADNeRFTorso.forward_torso with its gradient (section H, csrc/torso_train_kernel.cu); forward_torso calls it in
training mode.  `torso_sr_field` is the same for RADNeRFTorsowithSR.forward_torso (section I, csrc/torso_sr_train_kernel.cu).

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


# ------------------------------------------------------------------------------------------------ the head field
def _field_workspace(model, M):
    need = _capi.lib().gfpp_field_backward_workspace_bytes(M)
    if need == 0:
        raise _capi.GfppError(f"the training field does not support {M} points per call")
    dev = model.density_bitfield.device
    ws = model.__dict__.get("_field_ws")
    if ws is None or ws.numel() < need or ws.device != dev:
        ws = model.__dict__["_field_ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
    return ws


def _host_offsets(gp):
    """The grid's level offsets as a host int32 array, copied from the device once per offsets buffer (they never change in training)."""
    key = (gp.offsets.data_ptr(), gp.offsets._version)
    cached = gp.__dict__.get("_host_offsets")
    if cached is None or cached[0] != key:
        cached = gp.__dict__["_host_offsets"] = (key, np.ascontiguousarray(gp.offsets.detach().cpu().numpy().astype(np.int32)))
    return cached[1]


def _field_desc(model, code, keep):
    """The gfpp_model_desc fields section (G) reads -- grids, weights, code, cond_dim, bound, precision -- with no device-to-host copy."""
    d = _capi.ModelDesc()
    for name, gp in (("position_grid", model.position_embedder), ("ambient_grid", model.ambient_embedder)):
        g = getattr(d, name)
        lay = gp.layout
        emb = _cuda_f32(gp.embeddings.detach())
        off = _host_offsets(gp)
        keep += [emb, off]
        g.embeddings, g.offsets_host = emb.data_ptr(), off.ctypes.data
        g.input_dim, g.num_levels, g.base_resolution = lay.input_dim, lay.num_levels, lay.base_resolution
        g.log2_per_level_scale, g.gridtype, g.interp, g.align_corners = float(lay.S), lay.gridtype_id, lay.interp_id, int(lay.align_corners)
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
    dirs (the caller rejects inputs that require one)."""

    @staticmethod
    def forward(ctx, model, xyzs, dirs, cond_feat, code, *params):
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
        ws = _field_workspace(model, 0)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_field_forward(ctypes.byref(d), x.data_ptr(), dr.data_ptr(), M, c.data_ptr(), sigma.data_ptr(), color.data_ptr(),
                                                       amb.data_ptr(), ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_field_forward")
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
        g_sigma = torch.zeros(M, device=dev) if g_sigma is None else _cuda_f32(g_sigma)
        g_color = torch.zeros(M, 3, device=dev) if g_color is None else _cuda_f32(g_color)
        g_amb = torch.zeros(M, model.ambient_coord_dim, device=dev) if g_amb is None else _cuda_f32(g_amb)
        alloc = torch.zeros if M == 0 else torch.empty
        grad_w = [alloc(p.shape, dtype=torch.float32, device=dev) for p in params[:8]]
        g_pos = torch.zeros(params[8].shape, dtype=torch.float32, device=dev)
        g_tab = torch.zeros(params[9].shape, dtype=torch.float32, device=dev)
        g_cond = alloc(c.shape, dtype=torch.float32, device=dev)
        g_code = alloc(cd.shape, dtype=torch.float32, device=dev) if code_shape is not None else None
        keep = []
        d = _field_desc(model, cd if code_shape is not None else None, keep)
        ws = _field_workspace(model, M)
        ptrs = (ctypes.c_void_p * 8)(*[g.data_ptr() for g in grad_w])
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_field_backward(ctypes.byref(d), x.data_ptr(), dr.data_ptr(), M, c.data_ptr(), g_sigma.data_ptr(),
                                                        g_color.data_ptr(), g_amb.data_ptr(), ctypes.byref(ptrs), g_cond.data_ptr(),
                                                        None if g_code is None else g_code.data_ptr(), g_pos.data_ptr(), g_tab.data_ptr(),
                                                        ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_field_backward")
        grads = [g.to(p.dtype) for g, p in zip(grad_w + [g_pos, g_tab], params)]
        return (None, None, None, g_cond.view(cond_shape), None if g_code is None else g_code.view(code_shape), *grads)


field = _field.apply


# ------------------------------------------------------------------------------------------------ the torso field
def _torso_field_workspace(model, M):
    need = _capi.lib().gfpp_torso_field_workspace_bytes(M)
    if need == 0:
        raise _capi.GfppError(f"the torso training field does not support {M} points per call")
    dev = model.density_bitfield.device
    ws = model.__dict__.get("_torso_field_ws")
    if ws is None or ws.numel() < need or ws.device != dev:
        ws = model.__dict__["_torso_field_ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
    return ws


def _torso_field_desc(model, keep):
    """The gfpp_model_desc fields section (H) reads -- torso grid, the six torso weights, torso_code_dim, torso_shrink -- with no
    device-to-host copy."""
    d = _capi.ModelDesc()
    gp = model.torso_embedder
    lay = gp.layout
    emb = _cuda_f32(gp.embeddings.detach())
    off = _host_offsets(gp)
    keep += [emb, off]
    g = d.torso_grid
    g.embeddings, g.offsets_host = emb.data_ptr(), off.ctypes.data
    g.input_dim, g.num_levels, g.base_resolution = lay.input_dim, lay.num_levels, lay.base_resolution
    g.log2_per_level_scale, g.gridtype, g.interp, g.align_corners = float(lay.S), lay.gridtype_id, lay.interp_id, int(lay.align_corners)
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
        g_alpha = torch.zeros(M, device=dev) if g_alpha is None else _cuda_f32(g_alpha).reshape(-1)
        g_color = torch.zeros(M, 3, device=dev) if g_color is None else _cuda_f32(g_color)
        g_dx = torch.zeros(M, 2, device=dev) if g_dx is None else _cuda_f32(g_dx)
        alloc = torch.zeros if M == 0 else torch.empty
        grad_w = [alloc(p.shape, dtype=torch.float32, device=dev) for p in params[:6]]
        g_tab = torch.zeros(params[6].shape, dtype=torch.float32, device=dev)
        g_code = alloc(cd.shape, dtype=torch.float32, device=dev) if code_shape is not None else None
        keep = []
        d = _torso_field_desc(model, keep)
        ws = _torso_field_workspace(model, M)
        p_def = (ctypes.c_void_p * 3)(*[g.data_ptr() for g in grad_w[:3]])
        p_can = (ctypes.c_void_p * 3)(*[g.data_ptr() for g in grad_w[3:]])
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_field_backward(ctypes.byref(d), xy.data_ptr(), M, p6.data_ptr(),
                                                              None if code_shape is None else cd.data_ptr(), g_alpha.data_ptr(),
                                                              g_color.data_ptr(), g_dx.data_ptr(), ctypes.byref(p_def), ctypes.byref(p_can),
                                                              None if g_code is None else g_code.data_ptr(), g_tab.data_ptr(), ws.data_ptr(),
                                                              ws.numel(), _capi.stream_ptr(dev)), "gfpp_torso_field_backward")
        grads = [g.to(p.dtype) for g, p in zip(grad_w + [g_tab], params)]
        return (None, None, None, None if g_code is None else g_code.view(code_shape), *grads)


torso_field = _torso_field.apply


# ------------------------------------------------------------------------------------------------ the torso-SR field
def _torso_sr_field_workspace(model, M):
    need = _capi.lib().gfpp_torso_sr_field_workspace_bytes(M)
    if need == 0:
        raise _capi.GfppError(f"the torso-SR training field does not support {M} points per call")
    dev = model.density_bitfield.device
    ws = model.__dict__.get("_torso_sr_field_ws")
    if ws is None or ws.numel() < need or ws.device != dev:
        ws = model.__dict__["_torso_sr_field_ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
    return ws


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
    gp = model.torso_embedder
    lay = gp.layout
    ws = [_cuda_f32(p.detach()) for p in params]
    off = _host_offsets(gp)
    keep += ws + [off]
    g = d.torso_grid
    g.embeddings, g.offsets_host = ws[6].data_ptr(), off.ctypes.data
    g.input_dim, g.num_levels, g.base_resolution = lay.input_dim, lay.num_levels, lay.base_resolution
    g.log2_per_level_scale, g.gridtype, g.interp, g.align_corners = float(lay.S), lay.gridtype_id, lay.interp_id, int(lay.align_corners)
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
        g_alpha = torch.zeros(M, device=dev) if g_alpha is None else _cuda_f32(g_alpha).reshape(-1)
        g_color = torch.zeros(M, 3, device=dev) if g_color is None else _cuda_f32(g_color)
        g_dx = torch.zeros(M, 2, device=dev) if g_dx is None else _cuda_f32(g_dx)
        alloc = torch.zeros if M == 0 else torch.empty
        grads = [alloc(p.shape, dtype=torch.float32, device=dev) for p in params]
        grads[6] = torch.zeros(params[6].shape, dtype=torch.float32, device=dev)      # the table gradient is accumulated into
        g_code = alloc(cd.shape, dtype=torch.float32, device=dev) if code_shape is not None else None
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
