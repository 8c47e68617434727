"""oracle/torso_train.py -- TEST INFRASTRUCTURE (CPU checker; never imported by the product path).

RADNeRFTorso.forward_torso (modules/radnerfs/radnerf_torso.py:51-84) under torch autograd: the checker of libgfpp's training torso
field (gfpp.h section H).  The frequency encodings are the C restatement's (oracle/ops.py; x and the pose never require grad), the
torso grid is the autograd Function of oracle/field_train.py over the C restatement's grid_encode / grid_encode_dydx /
grid_encode_backward (the input gradient goes through dy_dx, as grid.py wires it), the dense layers are F.linear in the weights'
dtype (float32, or float64 for the reference gradients the tests measure against).

    alpha, color, dx = torso_forward(params, hparams, x, pose6, code)
    results = train_step(head_params, params, hparams, state, inputs, density_scale, max_steps)

train_step restates the training branch of RADNeRFTorso.render (radnerf_torso.py:86-199) with the head frozen: the head's training
render under no_grad (oracle/field_train.py), the grid_sample mask of density_grid_torso, forward_torso on the masked pixels, torso
over background, head over both, clamp.  eager_torso is the same field in eager PyTorch on the GPU (F.linear over a caller-chosen
grid_encode such as genefaceplusplus_b200.train_ops.grid_encode): the eager restatement that tests and tools/torso_train_bench.py
compare libgfpp's fused kernels with.

`params` maps the reference's state-dict names (torso_deform_net.net.{i}.weight, torso_canonicial_net.net.{i}.weight,
torso_embedder.embeddings / .offsets) to tensors; set requires_grad on the ones whose gradients are wanted.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import field_train as ft
from . import ops

TRAINABLE = ([f"torso_deform_net.net.{i}.weight" for i in range(3)] + [f"torso_canonicial_net.net.{i}.weight" for i in range(3)] +
             ["torso_embedder.embeddings"])
PLS_TORSO = float(np.exp2(np.log2(2048 / 16) / 15))   # the torso grid: tiled 2-D, desired resolution 2048 (radnerf_torso.py:31)


def torso_params(state, dtype=torch.float32):
    """The torso field's parameters from a state dict: trainable ones as fresh leaves that require grad (the table stays fp32, as
    in the reference), offsets as they are."""
    p = {}
    for k in TRAINABLE:
        t = state[k].detach().clone()
        p[k] = (t.to(dtype) if not k.endswith("embeddings") else t.float()).requires_grad_(True)
    p["torso_embedder.offsets"] = state["torso_embedder.offsets"]
    return p


def torso_forward(p, hp, x, pose6, code, trace=None):
    """(alpha [n,1], color [n,3], dx [n,2]) in the weights' dtype.  code: [1,dim] / [dim] or None.  trace: optional dict that
    receives the four ReLU pre-activations under "relu_pre" and shrink * x + dx (before the clamp) under "x_pre_clamp"."""
    dt = p["torso_deform_net.net.0.weight"].dtype
    interp_id = {"linear": 0, "smoothstep": 1}[hp["grid_interpolation_type"]]
    n = x.shape[0]
    xs = x.float() * hp["torso_shrink"]
    enc_x = ops.freq_encode(xs, 10).to(dt)
    enc_pose = ops.freq_encode(pose6.reshape(1, 6).float(), 4).to(dt)
    parts = [enc_x, enc_pose.repeat(n, 1)] + ([code.reshape(1, -1).to(dt).repeat(n, 1)] if code is not None else [])
    h = torch.cat(parts, dim=-1)
    pre = [] if trace is not None else None
    dx = ft._mlp(h, [p[f"torso_deform_net.net.{i}.weight"] for i in range(3)], pre)
    v = xs.to(dt) + dx
    x2 = v.clamp(-1, 1).float()
    feat = ft._GridEncode.apply((x2 + 1) / 2, p["torso_embedder.embeddings"], p["torso_embedder.offsets"], PLS_TORSO, 1, interp_id).to(dt)
    out = ft._mlp(torch.cat([feat, h], dim=-1), [p[f"torso_canonicial_net.net.{i}.weight"] for i in range(3)], pre)
    if trace is not None:
        trace["relu_pre"] = pre
        trace["x_pre_clamp"] = v.detach()
    return torch.sigmoid(out[..., :1]), torch.sigmoid(out[..., 1:]), dx


def tie_mask(trace, eps=1e-6):
    """Points within eps of a ReLU tie or of a clamp bound, where fp32 and float64 may take different branches, and points whose
    grid coordinate (x2 + 1) / 2 lies within eps of a cell boundary of some level, where dy_dx (the grid's input derivative) jumps."""
    v = trace["x_pre_clamp"]
    m = torch.zeros(v.shape[0], dtype=torch.bool)
    for t in trace["relu_pre"]:
        m |= (t.abs() < eps).any(-1)
    m |= ((v.abs() - 1).abs() < eps).any(-1)
    u = (v.clamp(-1, 1).double() + 1) / 2
    S = float(np.float32(np.log2(PLS_TORSO)))
    for l in range(16):
        scale = float(np.float32(np.exp2(np.float32(l * S)) * 16 - 1))
        p = u * scale + 0.5
        frac = p - torch.floor(p)
        m |= (torch.minimum(frac, 1 - frac) < eps * scale).any(-1)
    return m


def torso_mask(density_grid_torso, grid_size, bg_coords, thresh):
    """radnerf_torso.py:165-169."""
    occ = F.grid_sample(density_grid_torso.view(1, 1, grid_size, grid_size), bg_coords.float().view(1, -1, 1, 2), align_corners=True).view(-1)
    return occ > thresh


def head_train(head_params, hp, state, rays_o, rays_d, cond_feat, ind_code, density_scale, max_steps):
    """The head part of the torso training step (radnerf_torso.py:97-136, training branch) under no_grad: the premultiplied head
    image [N,3], weights_sum [N], nears, fars and depth."""
    bound = hp["bound"]
    cascade = 1 + int(np.ceil(np.log2(bound)))
    with torch.no_grad():
        ro, rd = rays_o.reshape(-1, 3).float().contiguous(), rays_d.reshape(-1, 3).float().contiguous()
        nears, fars = ops.near_far_from_aabb(ro, rd, state["aabb_train"], hp["min_near"])
        xyzs, dirs, deltas, rays, counter = ops.march_rays_train(ro, rd, bound, state["density_bitfield"], cascade, hp["grid_size"], nears, fars,
                                                                 dt_gamma=0.0, max_steps=max_steps)
        m = int(counter[0])
        m += 128 - m % 128
        sig, rgbs, amb = ft.field_forward(head_params, hp, xyzs[:m], dirs[:m], cond_feat, ind_code)
        ws, _, depth, image = ops.composite_rays_train_forward((density_scale * sig).float().contiguous(), rgbs.float().contiguous(),
                                                               amb.abs().sum(-1).float().contiguous(), deltas[:m].contiguous(), rays, 1e-4)
    return image, ws, nears, fars, depth


def composite(image, ws, mask, alpha_m, color_m, bg_color):
    """radnerf_torso.py:172-193 from the head image, the mask and the torso field on the masked pixels."""
    N = ws.shape[0]
    dt = alpha_m.dtype
    torso_alpha = torch.zeros(N, 1, dtype=dt)
    torso_color = torch.zeros(N, 3, dtype=dt)
    torso_alpha = torso_alpha.index_put((mask,), alpha_m)
    torso_color = torso_color.index_put((mask,), color_m)
    bg = torso_color * torso_alpha + bg_color.reshape(-1, 3).to(dt) * (1 - torso_alpha)
    rgb = (image.to(dt) + (1 - ws.to(dt)).unsqueeze(-1) * bg).clamp(0, 1)
    return {"torso_alpha_map": torso_alpha, "torso_rgb_map": bg, "rgb_map": rgb}


def train_step(head_params, p, hp, state, rays_o, rays_d, cond_feat, ind_code, bg_coords, pose6, torso_code, bg_color, density_scale, max_steps,
               mean_density_torso=0.0):
    """The training branch of RADNeRFTorso.render (radnerf_torso.py:86-199) on the CPU, gradients to the torso field only."""
    image, ws, nears, fars, depth = head_train(head_params, hp, state, rays_o, rays_d, cond_feat, ind_code, density_scale, max_steps)
    thr = min(hp["density_thresh_torso"], mean_density_torso)
    mask = torso_mask(state["density_grid_torso"], hp["grid_size"], bg_coords, thr)
    a, c, dx = torso_forward(p, hp, bg_coords.reshape(-1, 2)[mask], pose6, torso_code)
    res = composite(image, ws, mask, a, c, bg_color)
    res.update(weights_sum=ws, image=image, mask=mask, deform=dx)
    return res


def task_loss(res, gt, lambda_weights_entropy):
    """RADNeRFTorsoTask's loss for torso_train_mode 1 (tasks/radnerfs/radnerf_torso.py:92-106, 128-133): MSE of torso_rgb_map
    against the target bg_torso_img `gt` [N,3], plus lambda_weights_entropy times the mean binary entropy of the torso alpha."""
    mse = torch.mean((res["torso_rgb_map"].reshape(-1, 3) - gt.reshape(-1, 3).to(res["torso_rgb_map"].dtype)) ** 2)
    alphas = res["torso_alpha_map"].clamp(1e-5, 1 - 1e-5)
    entropy = torch.mean(-alphas * torch.log2(alphas) - (1 - alphas) * torch.log2(1 - alphas))
    return mse + lambda_weights_entropy * entropy


# ------------------------------------------------------------------------------------------------ inputs of tests/golden/train_torso.npz
GOLDEN_DS = 8.0          # density_scale of the head
GOLDEN_INDEX = 2         # training row of individual_embeddings / torso_individual_codes
GOLDEN_FRAME = 1
GOLDEN_MAX_STEPS = 16
GOLDEN_M = 3000          # points of part (a)
DEFORM_GAIN = 4.0        # torso_deform_net.net.2 is scaled so that |dx| reaches ~0.6 and shrink * x + dx leaves [-1, 1] near the edges
LAMBDA_WEIGHTS_ENTROPY = 1e-4   # egs/egs_bases/radnerf/base.yaml


def golden_scene():
    """The synthetic 32x32 May torso scene of the golden, with the deform net's output layer scaled by DEFORM_GAIN."""
    from genefaceplusplus_b200 import scene as scn
    sc = scn.Scene(H=32, W=32, T=4, torso=True, density_scale=GOLDEN_DS)
    sc.state["torso_deform_net.net.2.weight"] = sc.state["torso_deform_net.net.2.weight"] * DEFORM_GAIN
    return sc


def golden_points():
    """Part (a): GOLDEN_M points in [-1,1]^2 (a quarter of them within 0.1 of an edge) and the coefficients of the linear loss
    sum(alpha * ca) + sum(color * cc) + sum(dx * cd)."""
    g = torch.Generator().manual_seed(4321)
    x = torch.rand(GOLDEN_M, 2, generator=g) * 2 - 1
    q = GOLDEN_M // 4
    x[:q] = torch.sign(x[:q]) * (1 - 0.1 * torch.rand(q, 2, generator=g))
    return x, torch.randn(GOLDEN_M, 1, generator=g), torch.randn(GOLDEN_M, 3, generator=g), torch.randn(GOLDEN_M, 2, generator=g)


def golden_target(N):
    """Part (b): the seeded bg_torso_img target [N,3] of the MSE."""
    return torch.rand(N, 3, generator=torch.Generator().manual_seed(99))


# ------------------------------------------------------------------------------------------------ the step on libgfpp (GPU)
def gfpp_train_step(model, rays_o, rays_d, cond, bg_coords, poses, index, bg_color, max_steps, torso_field=None):
    """The training branch of RADNeRFTorso.render (radnerf_torso.py:86-199) assembled from libgfpp's training ops and a training-mode
    genefaceplusplus_b200 RADNeRFTorso `model` (mlp_precision "fp32"): the recipe README.md gives.  torso_field(x, poses, c) replaces
    model.forward_torso when given (the eager restatement of the tests and tools/torso_train_bench.py).  Returns the reference's
    result dict (torso_alpha_map, torso_rgb_map, rgb_map, weights_sum, deform)."""
    from genefaceplusplus_b200 import train_ops
    rays_o, rays_d, bg_coords = rays_o.reshape(-1, 3), rays_d.reshape(-1, 3), bg_coords.reshape(-1, 2)
    with torch.no_grad():   # the head is frozen
        nears, fars = train_ops.near_far_from_aabb(rays_o, rays_d, model.aabb_train, model.min_near)
        cond_feat = model.cal_cond_feat(cond)
        counter = model.step_counter[model.local_step % 16]
        counter.zero_()
        model.local_step += 1
        xyzs, dirs, deltas, rays = train_ops.march_rays_train(rays_o, rays_d, model.bound, model.density_bitfield, model.cascade, model.grid_size,
                                                              nears, fars, counter, model.mean_count, False, 128, False, 0, max_steps)
        sigmas, rgbs, ambient = model(xyzs, dirs, cond_feat, model.individual_embeddings[index])
        weights_sum, _, _, image = train_ops.composite_rays_train(model.density_scale * sigmas, rgbs, ambient.abs().sum(-1), deltas, rays)
    mask = model.torso_mask(bg_coords)
    N = rays_o.shape[0]
    torso_alpha = torch.zeros(N, 1, device=rays_o.device)
    torso_color = torch.zeros(N, 3, device=rays_o.device)
    field = torso_field or model.forward_torso
    alpha, color, deform = field(bg_coords[mask], poses, model.torso_individual_codes[index])
    torso_alpha[mask] = alpha
    torso_color[mask] = color
    bg = torso_color * torso_alpha + bg_color.reshape(-1, 3) * (1 - torso_alpha)
    rgb = (image + (1 - weights_sum).unsqueeze(-1) * bg).clamp(0, 1)
    return {"torso_alpha_map": torso_alpha, "torso_rgb_map": bg, "rgb_map": rgb, "weights_sum": weights_sum, "deform": deform}


# ------------------------------------------------------------------------------------------------ eager restatement (GPU)
def freq_encode_torch(x, degree):
    """[x, sin(2^f x), sin(2^f x + pi/2)]_f as freqencoder.cu:47-57 orders it, in torch (x never requires grad here)."""
    out = [x]
    for f in range(degree):
        s = x * (2.0 ** f)
        out += [torch.sin(s), torch.sin(s + math.pi / 2)]
    return torch.cat(out, dim=-1)


def eager_torso(model, P, x, pose6, code, grid_encode):
    """radnerf_torso.py:51-84 in eager PyTorch for a genefaceplusplus_b200 RADNeRFTorso `model` (layout, shrink) with parameters P
    (state-dict names); grid_encode has the signature of grid.py's grid_encode."""
    lay = model.torso_embedder.layout
    n = x.shape[0]
    xs = x * model.torso_shrink
    enc_x = freq_encode_torch(xs, 10)
    enc_pose = freq_encode_torch(pose6.reshape(1, 6), 4)
    parts = [enc_x, enc_pose.repeat(n, 1)] + ([code.reshape(1, -1).repeat(n, 1)] if code is not None else [])
    h = torch.cat(parts, dim=-1)
    dx = ft._mlp(h, [P[f"torso_deform_net.net.{i}.weight"] for i in range(3)])
    x2 = (xs + dx).clamp(-1, 1)
    feat = grid_encode((x2 + 1) / 2, P["torso_embedder.embeddings"], model.torso_embedder.offsets, lay.per_level_scale, 16, True, lay.gridtype_id,
                       False, lay.interp_id)
    out = ft._mlp(torch.cat([feat, h], dim=-1), [P[f"torso_canonicial_net.net.{i}.weight"] for i in range(3)])
    return torch.sigmoid(out[..., :1]), torch.sigmoid(out[..., 1:]), dx
