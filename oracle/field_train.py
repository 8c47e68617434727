"""oracle/field_train.py -- TEST INFRASTRUCTURE (CPU checker; never imported by the product path).

RADNeRF.forward (modules/radnerfs/radnerf.py:108-141) under torch autograd: the checker of libgfpp's training field (gfpp.h section G).
The grid encoders are autograd Functions over the C restatement of the reference's kernels (oracle/ops.py: grid_encode,
grid_encode_dydx, grid_encode_backward, as grid.py:24-88 wires them); trunc_exp has the reference's gradient (utils.py:36-47); the
dense layers are torch.nn.functional.linear in the weights' dtype (float32, or float64 for finite-difference checks).

    sigma, color, ambient_pos = field_forward(params, hparams, xyzs, dirs, cond_feat, individual_code)
    results = render_train(params, hparams, state, rays_o, rays_d, cond_feat, individual_code, bg_color, density_scale, max_steps)

render_train restates the training branch of NeRFRenderer.render (renderer.py:286-339, 385-398) around field_forward, with the C
restatement's marching and an autograd Function over its compositing.  eager_field is the same field in eager PyTorch on the GPU
(F.linear, a torch SH basis, grids through a caller-chosen grid_encode such as genefaceplusplus_b200.train_ops.grid_encode): the
eager restatement that tests and tools/train_step_bench.py compare libgfpp's fused kernels with.

`params` maps the reference's state-dict names (ambient_net.net.{i}.weight, sigma_net..., color_net..., position_embedder.embeddings /
.offsets, ambient_embedder.embeddings / .offsets) to tensors; set requires_grad on the ones whose gradients are wanted.
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch.autograd import Function

from . import ops


class _TruncExp(Function):
    """exp forward; backward g * exp(clamp(x, -15, 15))."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(-15, 15))


trunc_exp = _TruncExp.apply


class _GridEncode(Function):
    """inputs01 [B,D] in [0,1], embeddings [entries,2] -> [B, L*2] (fp32 C restatement); gradients w.r.t. the table and, when the
    inputs require one, w.r.t. the inputs through dy_dx."""

    @staticmethod
    def forward(ctx, inputs01, embeddings, offsets, per_level_scale, gridtype_id, interp_id):
        x = inputs01.detach().float().contiguous()
        e = embeddings.detach().float().contiguous()
        out = ops.grid_encode(x, e, offsets, per_level_scale, 16, gridtype_id, False, interp_id)
        dy_dx = ops.grid_encode_dydx(x, e, offsets, per_level_scale, 16, gridtype_id, False, interp_id) if inputs01.requires_grad else None
        ctx.save_for_backward(x, e, offsets)
        ctx.dy_dx = dy_dx
        ctx.meta = (per_level_scale, gridtype_id, interp_id, inputs01.dtype, embeddings.dtype)
        return out.to(embeddings.dtype)

    @staticmethod
    def backward(ctx, grad):
        x, e, offsets = ctx.saved_tensors
        pls, gridtype_id, interp_id, in_dtype, emb_dtype = ctx.meta
        ge, gi = ops.grid_encode_backward(grad.float().contiguous(), x, e, offsets, pls, 16, gridtype_id, False, interp_id, dy_dx=ctx.dy_dx)
        return (None if gi is None else gi.to(in_dtype)), ge.to(emb_dtype), None, None, None, None


def _grid(params, hp, name, x, bound, per_level_scale):
    gridtype_id = {"tiledgrid": 1, "hashgrid": 0}[hp["grid_type"]]
    interp_id = {"linear": 0, "smoothstep": 1}[hp["grid_interpolation_type"]]
    x01 = (x + bound) / (2 * bound)        # GridEncoder.forward (grid.py:152)
    return _GridEncode.apply(x01, params[f"{name}.embeddings"], params[f"{name}.offsets"], per_level_scale, gridtype_id, interp_id)


def _mlp(x, ws, pre=None):
    for i, w in enumerate(ws):
        x = F.linear(x, w)
        if i != len(ws) - 1:
            if pre is not None:
                pre.append(x.detach())
            x = F.relu(x)
    return x


def field_forward(params, hp, xyzs, dirs, cond_feat, individual_code, trace=None):
    """(sigma [N] raw, color [N,3], ambient_pos [N,A]) in the weights' dtype.  trace: optional dict that receives the pre-activations
    [N,128] of the five ReLUs (ambient 2, sigma 2, colour 1) under "relu_pre"."""
    bound = hp["bound"]
    pls = float(np.exp2(np.log2(hp["desired_resolution"] * bound / 16) / 15))
    pls_amb = float(np.exp2(np.log2(hp["desired_resolution"] / 16) / 15))
    n = xyzs.shape[0]
    dt = params["sigma_net.net.0.weight"].dtype
    cond = cond_feat.reshape(1, -1).repeat([n, 1])
    pos_feat = _grid(params, hp, "position_embedder", xyzs.float(), bound, pls).to(dt)
    pre = [] if trace is not None else None
    amb_logit = _mlp(torch.cat([pos_feat, cond], dim=1), [params[f"ambient_net.net.{i}.weight"] for i in range(3)], pre)
    amb = torch.tanh(amb_logit)
    amb_feat = _grid(params, hp, "ambient_embedder", amb, 1, pls_amb).to(dt)
    h = _mlp(torch.cat([pos_feat, amb_feat], dim=-1), [params[f"sigma_net.net.{i}.weight"] for i in range(3)], pre)
    sigma = trunc_exp(h[..., 0])
    geo = h[..., 1:]
    dfeat = ops.sh_encode(dirs, 4).to(dt)
    parts = [dfeat, geo] + ([individual_code.reshape(1, -1).repeat(n, 1)] if individual_code is not None else [])
    color = torch.sigmoid(_mlp(torch.cat(parts, dim=-1), [params[f"color_net.net.{i}.weight"] for i in range(2)], pre))
    if trace is not None:
        trace["relu_pre"] = pre
    return sigma, color, amb


TRAINABLE = ([f"ambient_net.net.{i}.weight" for i in range(3)] + [f"sigma_net.net.{i}.weight" for i in range(3)] +
             [f"color_net.net.{i}.weight" for i in range(2)] + ["position_embedder.embeddings", "ambient_embedder.embeddings"])


def field_params(state, dtype=torch.float32):
    """The field's parameters from a state dict: trainable ones as fresh leaves that require grad, offsets as they are."""
    p = {}
    for k in TRAINABLE:
        t = state[k].detach().clone()
        p[k] = (t.to(dtype) if not k.endswith("embeddings") else t.float()).requires_grad_(True)
    for k in ("position_embedder.offsets", "ambient_embedder.offsets"):
        p[k] = state[k]
    return p


class _CompositeTrain(Function):
    """composite_rays_train (raymarching.py:276-341) over the C restatement; grad_depth is not propagated, as there."""

    @staticmethod
    def forward(ctx, sigmas, rgbs, ambient, deltas, rays, T_thresh):
        s, r, a = sigmas.detach().float().contiguous(), rgbs.detach().float().contiguous(), ambient.detach().float().contiguous()
        ws, asum, depth, image = ops.composite_rays_train_forward(s, r, a, deltas, rays, T_thresh)
        ctx.save_for_backward(s, r, a, deltas, rays, ws, asum, image)
        ctx.T_thresh = T_thresh
        return ws, asum, depth, image

    @staticmethod
    def backward(ctx, g_ws, g_asum, g_depth, g_image):
        s, r, a, deltas, rays, ws, asum, image = ctx.saved_tensors
        gs, gr, ga = ops.composite_rays_train_backward(g_ws, g_asum, g_image, s, r, a, deltas, rays, ws, asum, image, ctx.T_thresh)
        return gs, gr, ga, None, None, None


def render_train(params, hp, state, rays_o, rays_d, cond_feat, individual_code, bg_color, density_scale, max_steps, dt_gamma=0.0):
    """The training branch of render() with mean_count 0 (all samples kept, truncated to the count rounded up to 128, as
    march_rays_train does), perturb False and composite_rays_train's default T_thresh."""
    bound = hp["bound"]
    cascade = 1 + int(np.ceil(np.log2(bound)))
    prefix = rays_o.shape[:-1]
    ro, rd = rays_o.reshape(-1, 3).float().contiguous(), rays_d.reshape(-1, 3).float().contiguous()
    nears, fars = ops.near_far_from_aabb(ro, rd, state["aabb_train"], hp["min_near"])
    xyzs, dirs, deltas, rays, counter = ops.march_rays_train(ro, rd, bound, state["density_bitfield"], cascade, hp["grid_size"], nears, fars,
                                                             dt_gamma=dt_gamma, max_steps=max_steps)
    m = int(counter[0])
    m += 128 - m % 128
    xyzs, dirs, deltas = xyzs[:m], dirs[:m], deltas[:m]
    sigmas, rgbs, ambient = field_forward(params, hp, xyzs, dirs, cond_feat, individual_code)
    sigmas = density_scale * sigmas
    ws, asum, depth, image = _CompositeTrain.apply(sigmas, rgbs, ambient.abs().sum(-1), deltas, rays, 1e-4)
    image = image + (1 - ws).unsqueeze(-1) * (1 if bg_color is None else bg_color)
    depth = torch.clamp(depth - nears, min=0) / (fars - nears)
    return {"weights_sum": ws, "ambient": asum, "position": xyzs, "rgb_map": image.view(*prefix, 3).clamp(0, 1), "depth_map": depth.view(*prefix)}


def sh4_torch(d):
    """Degree-4 real spherical harmonics (shencoder.cu:43-68) as torch ops."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    return torch.stack([torch.full_like(x, 0.28209479177387814), -0.48860251190291987 * y, 0.48860251190291987 * z, -0.48860251190291987 * x,
                        1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.94617469575755997 * z2 - 0.31539156525251999, -1.0925484305920792 * xz,
                        0.54627421529603959 * x2 - 0.54627421529603959 * y2, 0.59004358992664352 * y * (-3.0 * x2 + y2), 2.8906114426405538 * xy * z,
                        0.45704579946446572 * y * (1.0 - 5.0 * z2), 0.3731763325901154 * z * (5.0 * z2 - 3.0), 0.45704579946446572 * x * (1.0 - 5.0 * z2),
                        1.4453057213202769 * z * (x2 - y2), 0.59004358992664352 * x * (-x2 + 3.0 * y2)], dim=-1)


def eager_field(model, P, xyzs, dirs, cond_feat, code, grid_encode):
    """radnerf.py:108-141 in eager PyTorch for a genefaceplusplus_b200 RADNeRF `model` (layouts, bound) with parameters P (state-dict
    names); grid_encode has the signature of grid.py's grid_encode (inputs01, embeddings, offsets, per_level_scale, base_resolution,
    calc_grad_inputs, gridtype, align_corners, interpolation)."""
    lay_p, lay_a = model.position_embedder.layout, model.ambient_embedder.layout
    n = xyzs.shape[0]
    b = model.bound
    pos = grid_encode((xyzs + b) / (2 * b), P["position_embedder.embeddings"], model.position_embedder.offsets, lay_p.per_level_scale, 16, False,
                      lay_p.gridtype_id, False, lay_p.interp_id)
    h = _mlp(torch.cat([pos, cond_feat.reshape(1, -1).repeat(n, 1)], 1), [P[f"ambient_net.net.{i}.weight"] for i in range(3)])
    amb = torch.tanh(h)
    af = grid_encode((amb + 1) / 2, P["ambient_embedder.embeddings"], model.ambient_embedder.offsets, lay_a.per_level_scale, 16, True,
                     lay_a.gridtype_id, False, lay_a.interp_id)
    h = _mlp(torch.cat([pos, af], 1), [P[f"sigma_net.net.{i}.weight"] for i in range(3)])
    sigma = trunc_exp(h[:, 0])
    parts = [sh4_torch(dirs), h[:, 1:]] + ([code.reshape(1, -1).repeat(n, 1)] if code is not None else [])
    c = _mlp(torch.cat(parts, 1), [P[f"color_net.net.{i}.weight"] for i in range(2)])
    return sigma, torch.sigmoid(c), amb
