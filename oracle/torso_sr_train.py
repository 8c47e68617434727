"""oracle/torso_sr_train.py -- TEST INFRASTRUCTURE (CPU checker; never imported by the product path).

RADNeRFTorsowithSR.forward_torso (modules/radnerfs/radnerf_torso_sr.py:75-114) under torch autograd: the checker of libgfpp's
training torso-SR field (gfpp.h section I).  The frequency encodings are the C restatement's (oracle/ops.py; x and lm68 never require
grad), the torso grid is the autograd Function of oracle/field_train.py over the C restatement's grid ops (the input gradient goes
through dy_dx, as grid.py wires it), the dense layers -- the two torso MLPs and head_color_weights_encoder -- are F.linear in the
weights' dtype (float32, or float64 for the reference gradients the tests measure against).

    alpha, color, dx = torso_sr_forward(params, hparams, x, lm68, code, image, weights_sum)

eager_torso_sr is the same field in eager PyTorch on the GPU (F.linear over a caller-chosen grid_encode such as
genefaceplusplus_b200.train_ops.grid_encode): the eager restatement that tests and tools/torso_sr_train_bench.py compare libgfpp's
fused kernels with.

`params` maps the reference's state-dict names (torso_deform_net.net.{i}.weight, torso_canonicial_net.net.{i}.weight,
torso_embedder.embeddings / .offsets, head_color_weights_encoder.{0,2,4}.{weight,bias}) to tensors; set requires_grad on the ones
whose gradients are wanted.
"""
import torch
import torch.nn.functional as F

from . import field_train as ft
from . import ops
from . import torso_train as tt

TORSO = ([f"torso_deform_net.net.{i}.weight" for i in range(3)] + [f"torso_canonicial_net.net.{i}.weight" for i in range(3)] +
         ["torso_embedder.embeddings"])
HEAD_AWARE = [f"head_color_weights_encoder.{i}.{k}" for k in ("weight", "bias") for i in (0, 2, 4)]
PLS_TORSO = tt.PLS_TORSO
JAW = [5, 6, 7, 8, 9, 10, 11]


def trainable(head_aware):
    return TORSO + (HEAD_AWARE if head_aware else [])


def torso_sr_params(state, head_aware, dtype=torch.float32):
    """The field's parameters from a state dict: trainable ones as fresh leaves that require grad (the table stays fp32, as in the
    reference), offsets as they are."""
    p = {}
    for k in trainable(head_aware):
        t = state[k].detach().clone()
        p[k] = (t.to(dtype) if not k.endswith("embeddings") else t.float()).requires_grad_(True)
    p["torso_embedder.offsets"] = state["torso_embedder.offsets"]
    return p


def _head_aware(p, inp, pre):
    h = inp
    for j, i in enumerate((0, 2, 4)):
        h = F.linear(h, p[f"head_color_weights_encoder.{i}.weight"], p[f"head_color_weights_encoder.{i}.bias"])
        if j < 2:
            if pre is not None:
                pre.append(h.detach())
            h = F.leaky_relu(h, 0.02)
    return h


def torso_sr_forward(p, hp, x, lm68, code, image=None, weights_sum=None, trace=None):
    """(alpha [n,1], color [n,3], dx [n,2]) in the weights' dtype.  code: [1,dim] / [dim] or None; image [n,3] / weights_sum [n,1] or
    None (zeros).  trace: optional dict that receives the four ReLU and two LeakyReLU pre-activations under "relu_pre" and
    shrink * x + dx (before the clamp) under "x_pre_clamp" (the layout oracle/torso_train.tie_mask reads)."""
    dt = p["torso_deform_net.net.0.weight"].dtype
    interp_id = {"linear": 0, "smoothstep": 1}[hp["grid_interpolation_type"]]
    n = x.shape[0]
    xs = x.float() * hp["torso_shrink"]
    enc_x = ops.freq_encode(xs, 10).to(dt)
    jaw = lm68.reshape(1, 68, 2)[:, JAW].reshape(1, -1).float()
    enc_lm = ops.freq_encode(jaw, 4).to(dt)
    parts = [enc_x] + ([code.reshape(1, -1).to(dt).repeat(n, 1)] if code is not None else []) + [enc_lm.repeat(n, 1)]
    h = torch.cat(parts, dim=-1)
    pre = [] if trace is not None else None
    if hp["torso_head_aware"]:
        if image is None:
            image, weights_sum = torch.zeros(n, 3), torch.zeros(n, 1)
        inp = torch.cat([image.reshape(n, 3), weights_sum.reshape(n, 1)], dim=-1).to(dt)
        h = torch.cat([h, _head_aware(p, inp, pre)], dim=-1)
    dx = ft._mlp(h, [p[f"torso_deform_net.net.{i}.weight"] for i in range(3)], pre)
    v = xs.to(dt) + dx
    x2 = v.clamp(-1, 1).float()
    feat = ft._GridEncode.apply((x2 + 1) / 2, p["torso_embedder.embeddings"], p["torso_embedder.offsets"], PLS_TORSO, 1, interp_id).to(dt)
    out = ft._mlp(torch.cat([feat, h], dim=-1), [p[f"torso_canonicial_net.net.{i}.weight"] for i in range(3)], pre)
    if trace is not None:
        trace["relu_pre"] = pre
        trace["x_pre_clamp"] = v.detach()
    return torch.sigmoid(out[..., :1]), torch.sigmoid(out[..., 1:]), dx


def tie_mask(trace, eps=1e-6, relu_eps=1e-4):
    """oracle/torso_train.tie_mask with a wider margin for the ReLU / LeakyReLU kinks: the SR field's first layers sum ~200 inputs
    of magnitude up to ~10, so fp32 pre-activations computed in another summation order differ from float64 by up to ~1e-5 and
    take the other branch within that distance of zero.  Clamp bounds and grid cell boundaries keep the margin eps."""
    m = tt.tie_mask({"relu_pre": [], "x_pre_clamp": trace["x_pre_clamp"]}, eps)
    for t in trace["relu_pre"]:
        m |= (t.abs() < relu_eps).any(-1)
    return m


# ------------------------------------------------------------------------------------------------ inputs of tests/golden/train_torso_sr.npz
GOLDEN_INDEX = 2         # training row of torso_individual_codes
GOLDEN_FRAME = 1         # row of scene.lm68_sequence
GOLDEN_M = 3000          # points of each part
DEFORM_GAIN = 4.0        # torso_deform_net.net.2 is scaled so that shrink * x + dx leaves [-1, 1] near the edges (as train_torso.npz)
PARTS = {"a": dict(torso_head_aware=True), "b": dict(torso_head_aware=True), "c": dict(torso_head_aware=False, torso_individual_embedding_dim=0)}


BASE = dict(with_sr=True, add_eye_blink_cond=True, eye_blink_dim=4, smo_win_size=3)   # lm3d_radnerf_torso_sr.yaml (make_torso_sr_golden)


def golden_hparams(part):
    from genefaceplusplus_b200.config import may_hparams
    return may_hparams(**BASE, **PARTS[part])


def golden_state(hp):
    """The synthetic torso-SR state (scene.make_torso_sr_state) with the deform net's output layer scaled by DEFORM_GAIN."""
    from genefaceplusplus_b200 import scene as scn
    st = scn.make_torso_sr_state(hp)
    st["torso_deform_net.net.2.weight"] = st["torso_deform_net.net.2.weight"] * DEFORM_GAIN
    if hp["torso_individual_embedding_dim"] == 0:
        st.pop("torso_individual_codes", None)     # radnerf_torso_sr.py:27 registers no codes then
    return st


def golden_lm68():
    from genefaceplusplus_b200 import scene as scn
    return scn.lm68_sequence(4)[GOLDEN_FRAME].reshape(1, 136)


def golden_points(M=GOLDEN_M, seed=4321):
    """M points in [-1,1]^2 (a quarter of them within 0.1 of an edge), a premultiplied head image [M,3] with its alpha
    weights_sum [M,1], and the coefficients of the linear loss sum(alpha * ca) + sum(color * cc) + sum(dx * cd)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(M, 2, generator=g) * 2 - 1
    q = M // 4
    x[:q] = torch.sign(x[:q]) * (1 - 0.1 * torch.rand(q, 2, generator=g))
    ws = torch.rand(M, 1, generator=g)
    image = torch.rand(M, 3, generator=g) * ws
    return dict(x=x, image=image, weights_sum=ws, ca=torch.randn(M, 1, generator=g), cc=torch.randn(M, 3, generator=g),
                cd=torch.randn(M, 2, generator=g))


def linear_loss(a, c, dx, pts):
    return (a * pts["ca"].to(a.dtype)).sum() + (c * pts["cc"].to(c.dtype)).sum() + (dx * pts["cd"].to(dx.dtype)).sum()


# ------------------------------------------------------------------------------------------------ eager restatement (GPU)
def eager_torso_sr(model, P, x, lm68, code, image, weights_sum, grid_encode):
    """radnerf_torso_sr.py:75-114 in eager PyTorch for a genefaceplusplus_b200 RADNeRFTorsowithSR `model` (layout, shrink, head_aware)
    with parameters P (state-dict names); grid_encode has the signature of grid.py's grid_encode."""
    lay = model.torso_embedder.layout
    n = x.shape[0]
    xs = x * model.torso_shrink
    enc_x = tt.freq_encode_torch(xs, 10)
    enc_lm = tt.freq_encode_torch(lm68.reshape(1, 68, 2)[:, JAW].reshape(1, -1), 4)
    h = torch.cat([enc_x] + ([code.reshape(1, -1).repeat(n, 1)] if code is not None else []) + [enc_lm.repeat(n, 1)], dim=-1)
    if model.torso_head_aware:
        if image is None:
            image, weights_sum = torch.zeros(n, 3, device=x.device), torch.zeros(n, 1, device=x.device)
        h = torch.cat([h, _head_aware(P, torch.cat([image, weights_sum.reshape(n, 1)], dim=-1), None)], dim=-1)
    dx = ft._mlp(h, [P[f"torso_deform_net.net.{i}.weight"] for i in range(3)])
    x2 = (xs + dx).clamp(-1, 1)
    feat = grid_encode((x2 + 1) / 2, P["torso_embedder.embeddings"], model.torso_embedder.offsets, lay.per_level_scale, 16, True, lay.gridtype_id,
                       False, lay.interp_id)
    out = ft._mlp(torch.cat([feat, h], dim=-1), [P[f"torso_canonicial_net.net.{i}.weight"] for i in range(3)])
    return torch.sigmoid(out[..., :1]), torch.sigmoid(out[..., 1:]), dx


def model_params(model):
    """State-dict names -> the parameters of a genefaceplusplus_b200 RADNeRFTorsowithSR (for eager_torso_sr)."""
    P = {f"torso_deform_net.net.{i}.weight": model.torso_deform_net.net[i].weight for i in range(3)}
    P.update({f"torso_canonicial_net.net.{i}.weight": model.torso_canonicial_net.net[i].weight for i in range(3)})
    P["torso_embedder.embeddings"] = model.torso_embedder.embeddings
    if model.torso_head_aware:
        for i in (0, 2, 4):
            P[f"head_color_weights_encoder.{i}.weight"] = model.head_color_weights_encoder[i].weight
            P[f"head_color_weights_encoder.{i}.bias"] = model.head_color_weights_encoder[i].bias
    return P


def composite_and_loss(alpha, color, dx, mask, bg_color, gt, lambda_weights_entropy=1e-4, lambda_torso_deform=1e-3):
    """The torso part of RADNeRFTorsowithSR.render (radnerf_torso_sr.py:196-221) on the masked pixels and the torso terms of
    RADNeRFTorsoSRTask's loss before the SR losses (tasks/radnerfs/radnerf_torso_sr.py:154-161): MSE of torso_rgb_map against gt
    [N,3], lambda_weights_entropy times the mean binary entropy of the torso alpha, lambda_torso_deform times mean |deform|."""
    N = mask.shape[0]
    torso_alpha = torch.zeros(N, 1, device=alpha.device, dtype=alpha.dtype).index_put((mask,), alpha)
    torso_color = torch.zeros(N, 3, device=alpha.device, dtype=alpha.dtype).index_put((mask,), color)
    torso_bg = torso_color * torso_alpha + bg_color.reshape(-1, 3) * (1 - torso_alpha)
    mse = torch.mean((torso_bg - gt) ** 2)
    a = torso_alpha.clamp(1e-5, 1 - 1e-5)
    entropy = torch.mean(-a * torch.log2(a) - (1 - a) * torch.log2(1 - a))
    return mse + lambda_weights_entropy * entropy + lambda_torso_deform * dx.abs().mean()
