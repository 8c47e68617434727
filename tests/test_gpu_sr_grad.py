"""Gradients of the native SR head (train_ops.sr_head, include/gfpp.h section O) against float64 autograd of the torch path.

The native forward rounds the activations and the three GEMM layers' weights to fp16, as the reference's use_fp16 blocks do, and the
backward rounds the gradient operand of each GEMM to tf32.  So its gradients differ from float64 by those roundings carried through
the network.  The largest per-tensor relative L2 measured on an H100 SXM (80 GB, 700 W) over the cases below is 4.4e-2 (a noise
strength: one sum over 2^18 cancelling terms); BARS holds each tensor to about twice its own largest value.
Parameters whose float64 gradient is zero or absent get an absolute bar instead.
"""
import copy

import pytest
import torch

from genefaceplusplus_b200 import _capi, scene as scn
from genefaceplusplus_b200.superres import Superresolution

pytestmark = pytest.mark.gpu

BARS = {  # per tensor: about twice the largest relative L2 measured over CASES on an H100 SXM (80 GB, 700 W), at least 1e-5
    "block0.conv0.affine.bias": 1.4e-02, "block0.conv0.affine.weight": 1.4e-02, "block0.conv0.bias": 3.4e-02,
    "block0.conv0.noise_strength": 3.7e-02, "block0.conv0.weight": 7.8e-02, "block0.conv1.affine.bias": 2.5e-02,
    "block0.conv1.affine.weight": 2.5e-02, "block0.conv1.bias": 2.1e-02, "block0.conv1.noise_strength": 8.9e-02,
    "block0.conv1.weight": 2.3e-02, "block0.torgb.affine.bias": 6.0e-04, "block0.torgb.affine.weight": 6.0e-04,
    "block0.torgb.bias": 1.0e-05, "block0.torgb.weight": 5.6e-04, "block1.conv0.affine.bias": 3.5e-02,
    "block1.conv0.affine.weight": 3.5e-02, "block1.conv0.bias": 2.6e-02, "block1.conv0.noise_strength": 4.3e-02,
    "block1.conv0.weight": 2.9e-02, "block1.conv1.affine.bias": 1.8e-02, "block1.conv1.affine.weight": 1.8e-02,
    "block1.conv1.bias": 2.3e-02, "block1.conv1.noise_strength": 5.5e-02, "block1.conv1.weight": 4.1e-02,
    "block1.torgb.affine.bias": 8.3e-04, "block1.torgb.affine.weight": 8.3e-04, "block1.torgb.bias": 1.0e-05,
    "block1.torgb.weight": 7.7e-04, "input": 2.1e-02,
}
TORSO_STEP_REL = 2.2e-2   # torso-field gradients of the torso-SR step, native vs torch-path SR head: twice 1.1e-2 measured


def _state(loud):
    shapes = {k: tuple(v.shape) for k, v in Superresolution(channels=3).state_dict().items()}
    st = scn.synthetic_sr_state(shapes, seed=3)
    if loud:   # a quarter of the channels past the +256 clamp, a quarter on the leaky branch, a quarter with tiny weights
        for name in ("block0.conv0", "block0.conv1", "block1.conv0", "block1.conv1"):
            b, w = st[name + ".bias"].clone(), st[name + ".weight"].clone()
            b[0::4], b[1::4], b[2::4] = 320.0, -60.0, 0.0
            w[2::4] *= 1e-10
            st[name + ".bias"], st[name + ".weight"] = b, w
    return st


def _net(loud):
    net = Superresolution(channels=3)
    net.load_state_dict(_state(loud), strict=False)
    return net.cuda()


def _frames(F, R=256):
    a = scn.hashed_uniform(R * R * 3, 78, 1.0).reshape(R, R, 3) + 0.5
    pool = [a, 1.0 - a, torch.full_like(a, 0.25)]
    return torch.stack([pool[i % 3] for i in range(F)]).permute(0, 3, 1, 2).contiguous().cuda()


def _upstream(F):
    """A closed-form upstream gradient of the size a mean-reduced MSE over [F,3,512,512] gives."""
    return (scn.hashed_uniform(F * 3 * 512 * 512, 91, 1.0).reshape(F, 3, 512, 512) / (F * 3 * 512 * 512)).cuda()


def _ref64(net, rgb, noise_mode, raws):
    """float64 autograd of the torch path, with the native forward's own noise draws for 'random'."""
    ref = copy.deepcopy(net).double()
    ref.backend = "torch"
    if noise_mode == "random":
        for lay, r in zip(ref._layers(), raws):
            lay.noise_const = r.double()[:, None]          # per-frame planes, broadcast over channels
        noise_mode = "const"
    x = rgb.double().requires_grad_(True)
    w = torch.ones(ref.w_dim, dtype=torch.float64, device=x.device)
    feat, img = ref.block0(x, x, w, noise_mode)
    _, img = ref.block1(feat, img, w, noise_mode)
    return ref, x, img


def _native(net, rgb, noise_mode, seed=0):
    torch.manual_seed(seed)
    x = rgb.clone().requires_grad_(True)
    out = net(x, noise_mode=noise_mode)
    torch.manual_seed(seed)
    F = rgb.shape[0]
    raws = [torch.randn(F, r, r, device="cuda") for r in (256, 256, 512, 512)] if noise_mode == "random" else None
    return x, out, raws


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm().clamp_min(1e-300))


CASES = [("plain_f1_const", False, 1, "const"), ("loud_f1_none", True, 1, "none"), ("loud_f3_random", True, 3, "random"),
         ("plain_f3_random", False, 3, "random"), ("loud_f1_const", True, 1, "const")]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gradients_match_float64_autograd(case):
    _, loud, F, noise_mode = case
    net = _net(loud)
    with torch.no_grad():
        for lay in net._layers():                          # live noise terms, so the strengths' gradients are exercised
            lay.noise_strength.fill_(0.3)
    rgb = _frames(F)
    G = _upstream(F)
    x, out, raws = _native(net, rgb, noise_mode)
    (out * G).sum().backward()
    ref, x64, img64 = _ref64(net, rgb, noise_mode, raws)
    (img64 * G.double()).sum().backward()
    worst = {}
    pairs = [("input", x.grad, x64.grad)] + [(n, p.grad, q.grad) for (n, p), q in zip(net.named_parameters(), ref.parameters())]
    assert len(pairs) == 29 and sum(p.numel() for p in net.parameters()) == 271_229
    for name, g, g64 in pairs:
        assert g is not None, name
        if g64 is None or float(g64.norm()) == 0.0:          # e.g. the noise strengths with noise_mode 'none'
            assert float(g.abs().max()) < 1e-6, name
            continue
        worst[name] = _rel(g, g64)
    print(case[0], " ".join(f"{k}={v:.2e}" for k, v in sorted(worst.items(), key=lambda kv: -kv[1])))
    bad = {k: v for k, v in worst.items() if not v <= BARS[k]}
    assert not bad, bad


@pytest.mark.parametrize("noise_mode", ["const", "none"])
def test_forward_of_a_grad_call_is_bit_identical(noise_mode):
    net = _net(True)
    rgb = _frames(2)
    with torch.no_grad():
        ref = net(rgb, noise_mode=noise_mode)
    out = net(rgb.clone().requires_grad_(True), noise_mode=noise_mode)
    assert out.requires_grad
    assert torch.equal(out.detach(), ref)


def _abi_backward(grad_in, with_grad):
    """gfpp_sr_forward_train + gfpp_sr_backward called directly (the launch count is per host thread, and autograd runs the
    backward on its own thread); returns the backward's launch count."""
    import ctypes
    L = _capi.lib()
    net = _net(False)
    st = net._native_state()
    x = _frames(1).permute(0, 2, 3, 1).contiguous()
    out = torch.empty(1, 3, 512, 512, device="cuda")
    saved = torch.empty(L.gfpp_sr_train_workspace_bytes(1, 256), dtype=torch.uint8, device="cuda")
    _capi.check(L.gfpp_sr_forward_train(ctypes.byref(st["model"]), 1, 256, x.data_ptr(), None, 0, out.data_ptr(), saved.data_ptr(),
                                        saved.numel(), None), "gfpp_sr_forward_train")
    gd, keep = None, []
    if with_grad:
        gd = _capi.SrGrad()
        keep = [torch.empty(n, device="cuda") for n in (27 * 128, 128 * 1152, 256 * 1152, 64 * 576, 128, 128, 64, 64, 4, 384, 192, 3, 3)]
        gd.conv_in_w, gd.conv0_w, gd.up_w, gd.conv1_w = (t.data_ptr() for t in keep[:4])
        for i in range(4):
            gd.bias[i] = keep[4 + i].data_ptr()
        gd.noise_strength = keep[8].data_ptr()
        for i in range(2):
            gd.rgb_w[i], gd.rgb_b[i] = keep[9 + i].data_ptr(), keep[11 + i].data_ptr()
    gi = torch.empty_like(x) if grad_in else None
    ws = torch.empty(L.gfpp_sr_backward_workspace_bytes(1, 256), dtype=torch.uint8, device="cuda")
    _capi.check(L.gfpp_sr_backward(ctypes.byref(st["model"]), 1, 256, x.data_ptr(), saved.data_ptr(), saved.numel(), None, 0,
                                   _upstream(1).data_ptr(), None if gi is None else gi.data_ptr(), None if gd is None else ctypes.byref(gd),
                                   ws.data_ptr(), ws.numel(), None), "gfpp_sr_backward")
    n = L.gfpp_last_launch_count()
    torch.cuda.synchronize()
    return n


def test_frozen_parameters_run_dgrad_only():
    net = _net(False)
    for p in net.parameters():
        p.requires_grad_(False)
    x = _frames(1).requires_grad_(True)
    (net(x, noise_mode="const") * _upstream(1)).sum().backward()
    assert x.grad is not None and float(x.grad.abs().sum()) > 0
    assert all(p.grad is None for p in net.parameters())
    assert _abi_backward(grad_in=True, with_grad=False) == 7   # weight images, two toRGB stages, three dgrads, the input layer


def test_input_without_grad_skips_the_input_dgrad():
    net = _net(False)
    (net(_frames(1), noise_mode="const") * _upstream(1)).sum().backward()
    assert all(p.grad is not None for p in net.parameters())
    assert _abi_backward(grad_in=False, with_grad=True) == 6 + 3 * 2 + 2 + 4 * 3 + 2 * 2


def test_repeated_backward_is_bit_identical():
    net = _net(True)
    rgb, G = _frames(3), _upstream(3)
    runs = []
    for _ in range(2):
        net.zero_grad(set_to_none=True)
        x = rgb.clone().requires_grad_(True)
        (net(x, noise_mode="const") * G).sum().backward()
        runs.append([x.grad.clone()] + [p.grad.clone() for p in net.parameters()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_sr_phase_adam_steps_track_the_torch_path():
    """on_train_superresolution: the SR head alone, SR MSE against a 512^2 target, three Adam steps from the same state."""
    rgb = _frames(1)
    target = torch.nn.functional.interpolate(rgb, size=(512, 512), mode="bilinear", align_corners=False).clamp(0, 1) * 0.9
    nets, losses = [], []
    for backend in ("native", "torch"):
        net = _net(False)
        net.backend = backend
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        ls = []
        for _ in range(3):
            opt.zero_grad()
            loss = ((net(rgb, noise_mode="const") - target) ** 2).mean()
            loss.backward()
            opt.step()
            ls.append(float(loss.detach()))
        nets.append(net)
        losses.append(ls)
    print("losses native", losses[0], "torch", losses[1])
    for a, b in zip(*losses):
        assert abs(a - b) <= 1e-3 * abs(b)
    for (n, p), q in zip(nets[0].named_parameters(), nets[1].parameters()):
        assert float((p.detach() - q.detach()).norm()) <= 1e-3 * float(q.detach().norm()) + 1e-6, n


def test_torso_sr_step_with_the_native_sr_head():
    """One torso-SR training step (on_train_torso_nerf): torso_pass -> the torso losses + sr_torso_mse_loss, the task's SR loss
    (tasks/radnerfs/radnerf_torso_sr.py:163-168: MSE of clamp(sr_net(torso_rgb_map)) against the 512^2 target).  The torso field's
    and sr_net's gradients with the native SR head against the same step with the torch-path SR head."""
    import torch.nn.functional as Fn
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
    from oracle import torso_sr_train as tst, torso_train as tt
    hp = tst.golden_hparams("b")
    N = 256 * 256
    grads, losses = {}, {}
    for backend in ("native", "torch"):
        torch.manual_seed(5)
        m = RADNeRFTorsowithSR(hp)
        m.load_state_dict(tst.golden_state(hp), strict=False)
        m.density_scale, m.mlp_precision = tt.GOLDEN_DS, "fp32"
        m = m.cuda().train()
        m.sr_net.backend = backend
        g = torch.Generator(device="cuda").manual_seed(21)
        ws = torch.rand(N, generator=g, device="cuda")
        img = torch.rand(N, 3, generator=g, device="cuda") * ws[:, None]
        bgc = scn.get_bg_coords(256, 256).cuda().reshape(-1, 2)
        bg = torch.rand(1, N, 3, generator=g, device="cuda")
        gt = torch.rand(1, N, 3, generator=g, device="cuda")
        gt512 = torch.rand(1, 3, 512, 512, generator=g, device="cuda")
        row = torch.tensor([tst.GOLDEN_INDEX], device="cuda")
        code = m.torso_individual_codes[row] if m.torso_individual_embedding_dim else None
        res = m.torso_pass(img, ws, bgc, None, code, bg_color=bg, lm68=tst.golden_lm68().cuda())
        trgb = res["torso_rgb_map"]
        a = res["torso_alpha_map"].clamp(1e-5, 1 - 1e-5)
        loss = ((trgb - gt) ** 2).mean() + tt.LAMBDA_WEIGHTS_ENTROPY * (-a * torch.log2(a) - (1 - a) * torch.log2(1 - a)).mean() \
            + 1e-3 * res["deform"].abs().mean()
        sr = m.sr_net(trgb.reshape(1, 256, 256, 3).permute(0, 3, 1, 2), noise_mode="const").clamp(0, 1)
        loss = loss + Fn.mse_loss(sr, gt512)
        loss.backward()
        losses[backend] = float(loss.detach())
        grads[backend] = {k: p.grad.clone() for k, p in m.named_parameters()
                          if p.grad is not None and k.startswith(("torso_", "head_color_weights_encoder", "sr_net."))}
    assert grads["native"].keys() == grads["torch"].keys() and any(k.startswith("torso_") for k in grads["native"])
    print("\nlosses", losses)
    assert abs(losses["native"] - losses["torch"]) <= 1e-4 * abs(losses["torch"])
    # the torso field's gradients; sr_net's own are pinned against float64 above (the torch path's fp32 is no reference for the
    # noise strengths' cancelling sums)
    errs = {k: _rel(grads["native"][k], grads["torch"][k].double()) for k in grads["torch"]
            if float(grads["torch"][k].norm()) > 0 and not k.startswith("sr_net.")}
    print(" ".join(f"{k}={v:.2e}" for k, v in sorted(errs.items(), key=lambda kv: -kv[1])))
    for k, v in errs.items():
        assert v <= TORSO_STEP_REL, (k, v)
