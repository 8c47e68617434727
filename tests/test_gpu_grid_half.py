"""The grid encoder on half tables (gfpp.h section (L)) on the GPU, against the reference's own compiled half kernels
(oracle/_ref/_gridencoder, its at::Half instantiation) and the C checker (checkers/grid_half.c):

  * forward outputs, dy_dx and grad_inputs bit-equal to the reference's kernels and to the checker, for D = 2 and 3, tiled and
    hash, linear and smoothstep, B from 1 to 2^20 + 3;
  * the table gradient (f16x2 reductions in a free order) within K * 2^-11 * sum|terms| of the float64 sum of the checker's
    half-rounded terms, ours and the reference's alike;
  * the fp32 grid ops behind the shims unchanged;
  * end to end: oracle/render.py's restatement of the reference's host loop under torch.autocast(fp16), on the reference's
    extensions and on the shims, for the head and head+torso scenes at 512^2; and a restatement of grid.py's autograd Function
    in a head training step under autocast with a GradScaler, on both extension modules.
"""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.autograd import Function

from checkers import grid_half as gh
from genefaceplusplus_b200 import _capi, backend_shims
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import GridLayout

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def _load(name):
    so = os.path.join(REF, name, name + ".so")
    if not os.path.exists(so):
        pytest.skip(f"{so} not built (oracle/build_ref.py needs the reference sources)")
    spec = importlib.util.spec_from_file_location(name, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def ref_ge():
    return _load("_gridencoder")


@pytest.fixture(scope="module")
def our_ge():
    return backend_shims.make_modules()["_gridencoder"]


def _layout(D, gridtype, interp):
    return GridLayout(D, gridtype="hash" if gridtype == 0 else "tiled", interpolation="smoothstep" if interp else "linear",
                      desired_resolution=2048 if D == 3 else 256)


def _table(lay, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(lay.n_entries, 2, generator=g) * 0.1).half().cuda()


def _inputs(B, D, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, D, generator=g)
    if B > 8:
        x[0] = 0.0
        x[1] = 1.0
        x[2, 0] = -1e-3          # out of range: zeros, no gradient
        x[3, -1] = 1.0 + 1e-3
    return x.cuda()


def device_scales(lay):
    """The level scales the device computes (scale = fma(exp2f(l * S), H, -1)): torch's exp2 on the GPU is the same libdevice exp2f,
    and the fma is exact in float64 (a 24-bit mantissa times H <= 2^11, minus 1)."""
    e = torch.exp2(torch.arange(lay.num_levels, dtype=torch.float32, device="cuda") * float(lay.S)).cpu()
    return (e.double() * lay.base_resolution - 1.0).float()


def _bits(t):
    return t.contiguous().view(torch.int16)


def _run_forward(ge, x, emb, lay, dy_dx=True):
    B, D = x.shape
    L = lay.num_levels
    off = torch.from_numpy(lay.offsets).cuda()
    out = torch.empty(L, B, 2, dtype=torch.half, device="cuda")
    dd = torch.empty(B, L * D * 2, dtype=torch.half, device="cuda") if dy_dx else None
    ge.grid_encode_forward(x, emb, off, out, B, D, 2, L, float(lay.S), lay.base_resolution, dd, lay.gridtype_id, False, lay.interp_id)
    return out, dd


def _run_backward(ge, grad, x, emb, lay, dd):
    B, D = x.shape
    L = lay.num_levels
    off = torch.from_numpy(lay.offsets).cuda()
    gemb = torch.zeros_like(emb)
    gi = torch.zeros(B, D, dtype=torch.half, device="cuda") if dd is not None else None
    ge.grid_encode_backward(grad, x, emb, off, gemb, B, D, 2, L, float(lay.S), lay.base_resolution, dd, gi, lay.gridtype_id, False,
                            lay.interp_id)
    return gemb, gi


VARIANTS = [(D, gt, it) for D in (2, 3) for gt in (0, 1) for it in (0, 1)]


@pytest.mark.parametrize("B", [1, 4097, 390_784, 2 ** 20 + 3])
@pytest.mark.parametrize("D,gridtype,interp", VARIANTS)
def test_forward_dydx_and_input_grad_bit_equal(ref_ge, our_ge, D, gridtype, interp, B):
    lay = _layout(D, gridtype, interp)
    emb = _table(lay, 3 + D)
    x = _inputs(B, D, 100 + B % 97)
    out_r, dd_r = _run_forward(ref_ge, x, emb, lay)
    out_o, dd_o = _run_forward(our_ge, x, emb, lay)
    out_n, _ = _run_forward(our_ge, x, emb, lay, dy_dx=False)
    g = torch.Generator().manual_seed(7)
    grad = (torch.randn(lay.num_levels, B, 2, generator=g) * 0.05).half().cuda()
    _, gi_r = _run_backward(ref_ge, grad, x, emb, lay, dd_r)
    _, gi_o = _run_backward(our_ge, grad, x, emb, lay, dd_o)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out_o), _bits(out_r))
    assert torch.equal(_bits(out_n), _bits(out_r))
    assert torch.equal(_bits(dd_o), _bits(dd_r))
    assert torch.equal(_bits(gi_o), _bits(gi_r))
    # the checker on the first points, with the device's level scales
    n = min(B, 4097)
    xs = x[:n].cpu()
    oc, dc = gh.forward(xs, emb.cpu(), lay.offsets, lay.S, lay.base_resolution, gridtype=gridtype, interp=interp, dy_dx=True,
                        scales=device_scales(lay))
    gic = gh.input_grad(grad[:, :n].cpu(), dc)
    assert torch.equal(out_o[:, :n].cpu().float(), oc)
    assert torch.equal(dd_o[:n].cpu().float().reshape(dc.shape), dc)
    assert torch.equal(gi_o[:n].cpu().float(), gic)


@pytest.mark.parametrize("D,gridtype,interp", VARIANTS)
def test_table_gradient_within_the_rounding_bound(ref_ge, our_ge, D, gridtype, interp):
    """Each f16x2 add rounds its partial sum to half in an order the hardware picks: per entry, |result - exact sum of the rounded
    terms| <= K * 2^-11 * sum|terms| (+ K * 2^-25 where partial sums are subnormal), K the number of adds into the entry.  The
    reference's own kernel is held to the same bound."""
    B = 390_784
    lay = _layout(D, gridtype, interp)
    emb = _table(lay, 11 + D)
    x = _inputs(B, D, 5)
    g = torch.Generator().manual_seed(9)
    grad = (torch.randn(lay.num_levels, B, 2, generator=g) * 0.02).half().cuda()
    gr, _ = _run_backward(ref_ge, grad, x, emb, lay, None)
    go, _ = _run_backward(our_ge, grad, x, emb, lay, None)
    torch.cuda.synchronize()
    s, a, k = gh.table_grad(grad.cpu(), x.cpu(), lay.offsets, lay.n_entries, lay.S, lay.base_resolution, gridtype=gridtype, interp=interp,
                            scales=device_scales(lay))
    K = k.double()[:, None]
    bound = K * 2.0 ** -11 * a + K * 2.0 ** -25
    for name, got in (("ours", go), ("reference", gr)):
        err = (got.cpu().double() - s).abs()
        assert torch.isfinite(got).all(), name
        assert (err <= bound).all(), (name, float((err - bound).max()))
        assert (got.cpu()[k == 0] == 0).all(), name
        print(f"[table grad D={D} gridtype={gridtype} interp={interp}] {name}: max err / bound {float((err / bound.clamp(min=1e-30)).max()):.3f}, "
              f"max err {float(err.max()):.3e}, entries hit {int((k > 0).sum())}")


def test_fp32_calls_take_the_fp32_ops(our_ge):
    """The fp32 shims are the calls they were: bit-identical to the fp32 C-ABI entry points (sections A and D) called directly."""
    L = _capi.lib()
    S = _capi.stream_ptr
    lay = _layout(3, 1, 0)
    B, D = 4097, 3
    emb = _table(lay, 1).float()
    x = _inputs(B, D, 2)
    off = torch.from_numpy(lay.offsets).cuda()
    out, dd = torch.empty(16, B, 2, device="cuda"), torch.empty(B, 16 * D * 2, device="cuda")
    our_ge.grid_encode_forward(x, emb, off, out, B, D, 2, 16, float(lay.S), 16, dd, 1, False, 0)
    out2, dd2 = torch.empty_like(out), torch.empty_like(dd)
    P = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    offs = np.ascontiguousarray(lay.offsets)
    _capi.check(L.gfpp_grid_encode_forward_dydx(P(x), P(emb), offs.ctypes.data_as(ctypes.c_void_p), P(out2), B, D, 2, 16, float(lay.S), 16,
                                                P(dd2), 1, 0, 0, S()), "forward")
    grad = torch.randn(16, B, 2, device="cuda") * 0.05
    ge1, gi1 = torch.zeros_like(emb), torch.zeros(B, D, device="cuda")
    our_ge.grid_encode_backward(grad, x, emb, off, ge1, B, D, 2, 16, float(lay.S), 16, dd, gi1, 1, False, 0)
    ge2, gi2 = torch.zeros_like(emb), torch.zeros(B, D, device="cuda")
    _capi.check(L.gfpp_grid_encode_backward(P(grad), P(x), P(emb), offs.ctypes.data_as(ctypes.c_void_p), P(ge2), B, D, 2, 16, float(lay.S), 16,
                                            P(dd2), P(gi2), 1, 0, 0, S()), "backward")
    torch.cuda.synchronize()
    assert torch.equal(out, out2) and torch.equal(dd, dd2) and torch.equal(gi1, gi2)
    assert (ge1 - ge2).abs().max().item() <= 1e-6 * ge2.abs().max().item()      # float2 reductions in a free order
    with pytest.raises(RuntimeError):                                           # an fp32 table with half outputs
        our_ge.grid_encode_forward(x, emb, off, out.half(), B, D, 2, 16, float(lay.S), 16, None, 1, False, 0)


# ------------------------------------------------------------------------------------------------ end to end: inference under autocast
def _shim_ref_ops():
    """oracle/gpu_ref_ops (the reference's wrappers restated) with its extension modules replaced by backend_shims.make_modules()."""
    from oracle import gpu_ref_ops
    spec = importlib.util.spec_from_file_location("gpu_shim_ops", gpu_ref_ops.__file__)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod._mods.update(backend_shims.make_modules())
    return mod


def _cmp(a, b):
    d = (a.float() - b.float()).abs().reshape(-1, 3).max(-1).values
    mse = ((a.double() - b.double()) ** 2).mean().item()
    return {"max_abs": d.max().item(), "n_over_1e-3": int((d > 1e-3).sum().item()), "n_pixels": d.numel(),
            "psnr": 999.0 if mse == 0 else 10 * math.log10(1.0 / mse)}


@pytest.mark.parametrize("torso", [False, True])
def test_reference_host_loop_under_autocast_on_the_shims(torso):
    for n in ("_raymarching_face", "_gridencoder", "_shencoder", "_freqencoder"):
        _load(n)
    from oracle import gpu_ref_ops
    from oracle.render import OracleModel
    dev = torch.device("cuda", torch.cuda.current_device())
    sc = scn.Scene(H=512, W=512, T=2, torso=torso, density_scale=8.0)
    fi = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc.frame_inputs(1).items()}
    imgs = {}
    for name, backend in (("reference", gpu_ref_ops), ("shims", _shim_ref_ops())):
        m = OracleModel(sc.state, sc.hparams, backend=backend, device=dev, collect_stats=False)
        m.density_scale = 8.0
        with torch.autocast("cuda", dtype=torch.float16):
            imgs[name] = m.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"],
                                  T_thresh=sc.T_thresh, **sc.hparams)["rgb_map"].float().reshape(-1, 3)
    torch.cuda.synchronize()
    c = _cmp(imgs["shims"], imgs["reference"])
    print(f"[autocast render 512^2 torso={torso}] shims vs reference extensions: {c}")
    assert torch.isfinite(imgs["shims"]).all()
    # the half grid lookups are bit-exact; the marching ops differ by cell flips (the reference's FMA contraction, one boundary
    # sample more or less, tools/ref_gpu_baseline.py): measured 1 pixel over 1e-3 and 90 / 94 dB (head / head+torso) on the H100
    assert c["n_over_1e-3"] <= 64 and c["psnr"] >= 70.0, c


# ------------------------------------------------------------------------------------------------ end to end: training under autocast
def grid_encode_fn(ext):
    """grid.py:24-88 restated, over the extension module `ext`: custom_fwd, half tables under autocast when C is even, a half
    backward; the input gradient comes back in the inputs' dtype."""

    class _GridEncode(Function):
        @staticmethod
        @torch.amp.custom_fwd(device_type="cuda")
        def forward(ctx, inputs, embeddings, offsets, per_level_scale, base_resolution, calc_grad_inputs=False, gridtype=0,
                    align_corners=False, interpolation=0):
            inputs = inputs.contiguous()
            B, D = inputs.shape
            L = offsets.shape[0] - 1
            C = embeddings.shape[1]
            S = np.log2(per_level_scale)
            H = base_resolution
            if torch.is_autocast_enabled() and C % 2 == 0:
                embeddings = embeddings.to(torch.half)
            outputs = torch.empty(L, B, C, device=inputs.device, dtype=embeddings.dtype)
            dy_dx = torch.empty(B, L * D * C, device=inputs.device, dtype=embeddings.dtype) if calc_grad_inputs else None
            ext.grid_encode_forward(inputs, embeddings, offsets, outputs, B, D, C, L, S, H, dy_dx, gridtype, align_corners, interpolation)
            outputs = outputs.permute(1, 0, 2).reshape(B, L * C)
            ctx.save_for_backward(inputs, embeddings, offsets, dy_dx)
            ctx.dims = [B, D, C, L, S, H, gridtype, interpolation]
            ctx.align_corners = align_corners
            return outputs

        @staticmethod
        @torch.amp.custom_bwd(device_type="cuda")
        def backward(ctx, grad):
            inputs, embeddings, offsets, dy_dx = ctx.saved_tensors
            B, D, C, L, S, H, gridtype, interpolation = ctx.dims
            grad = grad.view(B, L, C).permute(1, 0, 2).contiguous()
            grad_embeddings = torch.zeros_like(embeddings)
            grad_inputs = torch.zeros_like(inputs, dtype=embeddings.dtype) if dy_dx is not None else None
            ext.grid_encode_backward(grad, inputs, embeddings, offsets, grad_embeddings, B, D, C, L, S, H, dy_dx, grad_inputs, gridtype,
                                     ctx.align_corners, interpolation)
            if dy_dx is not None:
                grad_inputs = grad_inputs.to(inputs.dtype)
            return grad_inputs, grad_embeddings, None, None, None, None, None, None, None

    return _GridEncode.apply


def _field(model, P, xyzs, dirs, cond_feat, code, grid_encode):
    """RADNeRF.forward (radnerf.py:108-141) as the reference writes it for amp: the ambient logit in fp32 (.float()), trunc_exp on fp32."""
    from oracle import field_train as ft
    lp, la = model.position_embedder.layout, model.ambient_embedder.layout
    n, b = xyzs.shape[0], model.bound
    pos = grid_encode((xyzs + b) / (2 * b), P["position_embedder.embeddings"], model.position_embedder.offsets, lp.per_level_scale, 16,
                      False, lp.gridtype_id, False, lp.interp_id)
    x = torch.cat([pos, cond_feat.reshape(1, -1).repeat(n, 1)], 1)
    for i in range(3):
        x = F.linear(x, P[f"ambient_net.net.{i}.weight"])
        x = F.relu(x) if i < 2 else x
    amb = torch.tanh(x.float())
    af = grid_encode((amb + 1) / 2, P["ambient_embedder.embeddings"], model.ambient_embedder.offsets, la.per_level_scale, 16, True,
                     la.gridtype_id, False, la.interp_id)
    h = torch.cat([pos, af], 1)
    for i in range(3):
        h = F.linear(h, P[f"sigma_net.net.{i}.weight"])
        h = F.relu(h) if i < 2 else h
    sigma = ft.trunc_exp(h[:, 0].float())
    c = torch.cat([ft.sh4_torch(dirs), h[:, 1:], code.reshape(1, -1).repeat(n, 1)], 1)
    for i in range(2):
        c = F.linear(c, P[f"color_net.net.{i}.weight"])
        c = F.relu(c) if i < 1 else c
    return sigma, torch.sigmoid(c.float()), amb


def _step_setup(H, W):
    from genefaceplusplus_b200 import train_ops
    from genefaceplusplus_b200.renderer import RADNeRF
    sc = scn.Scene(H=H, W=W, T=4, torso=False, density_scale=8.0)
    model = RADNeRF(sc.hparams)
    model.load_state_dict(sc.state, strict=True)
    model = model.cuda()
    if H == 32:
        G = np.load(os.path.join(ROOT, "tests", "golden", "train_head.npz"))
        ro, rd, bg = (torch.from_numpy(G[k]).reshape(-1, 3).cuda() for k in ("rays_o", "rays_d", "bg_color"))
        cf = torch.from_numpy(G["cond_feat"]).cuda()
    else:
        fi = sc.frame_inputs(2)
        ro, rd, bg = fi["rays_o"].reshape(-1, 3).cuda(), fi["rays_d"].reshape(-1, 3).cuda(), fi["bg_color"].reshape(-1, 3).cuda()
        cf = (torch.randn(64, generator=torch.Generator().manual_seed(4)) * 0.5).cuda()
    ro, rd = ro.contiguous(), rd.contiguous()
    nears, fars = train_ops.near_far_from_aabb(ro, rd, sc.state["aabb_train"].cuda(), sc.hparams["min_near"])
    xyzs, dirs, deltas, rays = train_ops.march_rays_train(ro, rd, 1.0, sc.state["density_bitfield"].cuda(), 1, sc.hparams["grid_size"], nears,
                                                          fars, None, -1, False, 128, False, 0.0, 16)
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(6)).cuda()
    return sc, model, (xyzs, dirs, deltas, rays), cf, bg, target


def _train(sc, model, samples, cf, bg, target, ext, steps):
    """`steps` Adam steps of the head field under autocast with a GradScaler; returns (losses, maps and gradients of the first step,
    scales)."""
    from genefaceplusplus_b200 import train_ops
    from oracle import field_train as ft
    xyzs, dirs, deltas, rays = samples
    P = {k: v.cuda() for k, v in ft.field_params(sc.state).items()}
    for k in ft.TRAINABLE:
        P[k] = P[k].detach().requires_grad_(True)
    code = sc.state["individual_embeddings"][2].cuda().clone().requires_grad_(True)
    opt = torch.optim.Adam([P[k] for k in ft.TRAINABLE] + [code], lr=1e-3, betas=(0.9, 0.99), eps=1e-15)
    scaler = torch.amp.GradScaler("cuda")
    enc = grid_encode_fn(ext)
    losses, first, scales = [], None, []
    for it in range(steps):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            sigma, color, amb = _field(model, P, xyzs, dirs, cf, code, enc)
            ws, asum, _, image = train_ops.composite_rays_train(8.0 * sigma, color, amb.abs().sum(-1), deltas, rays, 1e-4)
            rgb = image + (1 - ws).unsqueeze(-1) * bg
            loss = F.mse_loss(rgb, target) + 1e-3 * asum.mean()
        scale0 = scaler.get_scale()
        scaler.scale(loss).backward()
        if it == 0:
            first = {"rgb_map": rgb.detach().clone(), "weights_sum": ws.detach().clone(), "ambient": asum.detach().clone()}
            first.update({"grad." + k: (P[k].grad.detach().float() / scale0).clone() for k in ft.TRAINABLE})
            first["grad.individual_code"] = (code.grad.detach() / scale0).clone()
        scaler.step(opt)
        scaler.update()
        scales.append((scale0, scaler.get_scale()))
        losses.append(loss.item())
    return losses, first, scales


@pytest.mark.parametrize("size", [32, 256])
def test_training_steps_under_autocast_on_both_modules(ref_ge, our_ge, size):
    """One head training step on the train_head.npz rays (32^2) and one at 65 536 rays (256^2), then 20 Adam steps, under autocast
    with a GradScaler: grid.py's Function over the reference's _gridencoder and over the shim's.  Marching and compositing are
    libgfpp's fp32 training ops in both runs, so the grid encoder is the only difference."""
    sc, model, samples, cf, bg, target = _step_setup(size, size)
    steps = 20 if size == 32 else 1
    lr, fr, sr = _train(sc, model, samples, cf, bg, target, ref_ge, steps)
    lo, fo, so = _train(sc, model, samples, cf, bg, target, our_ge, steps)
    torch.cuda.synchronize()
    print(f"[train {size}^2: {samples[0].shape[0]} samples] losses reference {lr[0]:.6f} -> {lr[-1]:.6f}, shims {lo[0]:.6f} -> {lo[-1]:.6f}")
    for s0, s1 in sr + so:
        assert s1 >= s0, "the GradScaler skipped a step (inf/nan in the half gradients)"
    worst = {}
    for k, v in fr.items():
        e = (fo[k] - v).abs().max().item() / max(v.abs().max().item(), 1e-30)
        worst[k] = e
    print(f"[train {size}^2] first-step relative max difference shims vs reference: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    # the forward and every gradient upstream of the grids are bit-identical (the half kernels are); the two table gradients
    # differ by the order of their f16x2 reductions, as two runs of the reference's own kernel do
    _, fr2, _ = _train(sc, model, samples, cf, bg, target, ref_ge, 1)
    spread = {k: (fr2[k] - fr[k]).abs().max().item() / max(fr[k].abs().max().item(), 1e-30) for k in fr if k.endswith("embeddings")}
    print(f"[train {size}^2] reference run to run, tables: " + ", ".join(f"{k} {v:.2e}" for k, v in spread.items()))
    for k, e in worst.items():
        if k.endswith("embeddings"):
            assert e <= 0.1, (k, e)     # relative to the largest entry; measured 4.2e-2 (position) at 65 536 rays
        else:
            assert e == 0.0, (k, e)
    if steps > 1:
        rel = max(abs(a - b) / abs(b) for a, b in zip(lo, lr))
        print(f"[train {size}^2] 20 Adam steps: max relative loss difference {rel:.2e}")
        assert lo[-1] < lo[0] and rel <= 1e-2, (rel, lo, lr)
