"""CPU checks of the checker's TRAINING-side restatement (oracle/native_ops.c, second half; SURVEY 8(f) rank 4).

The reference ships these ops as CUDA only and has no tests for them, so the restatement is pinned here through properties that
do not need the reference: the train marcher against the (reference-pinned) inference marcher, compositing backward against
autograd of the rendering formula, the grid backward as the exact adjoint of the (reference-pinned) forward, dy_dx against finite
differences, Morton / bit-packing identities.  On the GPU the same functions are pinned against the reference's own kernels
(tests/test_gpu_train_ops.py)."""
import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import GridLayout


def _rays(oracle_ops, H=40, T_frame=1):
    sc = scn.Scene(H=H, W=H, T=2, torso=False)
    fi = sc.frame_inputs(T_frame)
    ro, rd = fi["rays_o"].view(-1, 3).contiguous(), fi["rays_d"].view(-1, 3).contiguous()
    nears, fars = oracle_ops.near_far_from_aabb(ro, rd, sc.state["aabb_infer"], 0.05)
    return sc, ro, rd, nears, fars


@pytest.mark.parametrize("max_steps,dt_gamma", [(16, 1 / 256), (64, 0.0)])
def test_train_marcher_equals_the_inference_marcher(oracle_ops, max_steps, dt_gamma):
    sc, ro, rd, nears, fars = _rays(oracle_ops)
    bits = sc.state["density_bitfield"]
    N = ro.shape[0]
    xyzs, dirs, deltas, rays, counter = oracle_ops.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, dt_gamma=dt_gamma, max_steps=max_steps)
    assert counter.tolist() == [int(rays[:, 2].sum()), N]
    assert torch.equal(rays[:, 0], torch.arange(N, dtype=torch.int32))
    assert torch.equal(rays[:, 1].long(), torch.cumsum(rays[:, 2].long(), 0) - rays[:, 2].long())          # exclusive prefix sum, ray order
    # one inference round with n_step = max_steps from t = near emits the same samples (raymarching.cu:827-929 vs :464-517)
    alive = torch.arange(N, dtype=torch.int32)
    x2, d2, l2 = oracle_ops.march_rays(N, max_steps, alive, nears.clone(), ro, rd, 1.0, bits, 1, 128, nears, fars, -1, False, dt_gamma, max_steps)
    x2, l2 = x2.view(N, max_steps, 3), l2.view(N, max_steps, 2)
    cnt = (l2[:, :, 0] > 0).sum(1).int()
    assert torch.equal(cnt, rays[:, 2])
    assert rays[:, 2].max().item() > 4 and (rays[:, 2] == 0).any()
    for n in torch.nonzero(rays[:, 2] > 0).view(-1)[::37].tolist():
        o, k = int(rays[n, 1]), int(rays[n, 2])
        assert torch.equal(xyzs[o:o + k], x2[n, :k]) and torch.equal(deltas[o:o + k], l2[n, :k])
        assert torch.equal(dirs[o:o + k], rd[n].expand(k, 3))
    # overflow: rays that do not fit into M keep their row but write nothing
    M = int(counter[0]) // 2
    xs, _, ls, rs, _ = oracle_ops.march_rays_train(ro, rd, 1.0, bits, 1, 128, nears, fars, M=M, dt_gamma=dt_gamma, max_steps=max_steps)
    assert torch.equal(rs, rays)
    fit = (rays[:, 1] + rays[:, 2]) <= M
    last = int(torch.nonzero(fit & (rays[:, 2] > 0)).max())
    end = int(rays[last, 1] + rays[last, 2])
    assert torch.equal(xs[:end], xyzs[:end]) and ls[end:].abs().sum().item() == 0


def _segments(N=200, seed=0, max_len=24):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, max_len, (N,), generator=g, dtype=torch.int32)
    lens[::7] = 0
    lens[3] = 70                                                                                           # longer than two warps' trips
    offs = torch.cumsum(lens.long(), 0) - lens.long()
    perm = torch.randperm(N, generator=g).int()                                                            # rays[:,0] is a permutation
    rays = torch.stack([perm, offs.int(), lens], 1).contiguous()
    M = int(lens.sum())
    sig = torch.rand(M, generator=g) * 6
    rgb = torch.rand(M, 3, generator=g)
    amb = torch.rand(M, generator=g)
    dt = torch.rand(M, generator=g) * 0.05 + 0.01
    deltas = torch.stack([dt, torch.rand(M, generator=g) * 3 + 2], 1).contiguous()
    return rays, M, sig, rgb, amb, deltas


def _formula(sig, rgb, amb, deltas, rays, T_thresh):
    """The rendering integral in differentiable torch (double), with the reference's early break."""
    N = rays.shape[0]
    ws, asum, depth, image = torch.zeros(N, dtype=sig.dtype), torch.zeros(N, dtype=sig.dtype), torch.zeros(N, dtype=sig.dtype), torch.zeros(N, 3, dtype=sig.dtype)
    ws, asum, depth, image = list(ws), list(asum), list(depth), [image[i] for i in range(N)]
    for n in range(N):
        idx, o, k = int(rays[n, 0]), int(rays[n, 1]), int(rays[n, 2])
        T = torch.ones((), dtype=sig.dtype)
        w_, a_, d_, c_ = 0, 0, 0, 0
        for s in range(o, o + k):
            alpha = 1 - torch.exp(-sig[s] * deltas[s, 0])
            w = alpha * T
            w_, a_, d_, c_ = w_ + w, a_ + amb[s], d_ + w * deltas[s, 1], c_ + w * rgb[s]
            T = T * (1 - alpha)
            if T.item() < T_thresh:
                break
        if k:
            ws[idx], asum[idx], depth[idx], image[idx] = w_, a_, d_, c_
    return torch.stack([torch.as_tensor(v, dtype=sig.dtype) for v in ws]), torch.stack([torch.as_tensor(v, dtype=sig.dtype) for v in asum]), \
        torch.stack([torch.as_tensor(v, dtype=sig.dtype) for v in depth]), torch.stack([v if torch.is_tensor(v) and v.dim() else torch.zeros(3, dtype=sig.dtype) for v in image])


@pytest.mark.parametrize("T_thresh", [1e-4, 0.2])
def test_composite_train_forward_and_backward_match_autograd_of_the_formula(oracle_ops, T_thresh):
    rays, M, sig, rgb, amb, deltas = _segments()
    ws, asum, depth, image = oracle_ops.composite_rays_train_forward(sig, rgb, amb, deltas, rays, T_thresh)
    sd, rd_, ad = sig.double().requires_grad_(), rgb.double().requires_grad_(), amb.double().requires_grad_()
    fw, fa, fd, fi = _formula(sd, rd_, ad, deltas.double(), rays, T_thresh)
    for got, ref in ((ws, fw), (asum, fa), (depth, fd), (image, fi)):
        assert (got.double() - ref.detach()).abs().max().item() < 2e-5
    g = torch.Generator().manual_seed(9)
    gws, gas, gim = torch.randn(rays.shape[0], generator=g), torch.randn(rays.shape[0], generator=g), torch.randn(rays.shape[0], 3, generator=g)
    # the reference does not propagate the depth gradient (raymarching.py:303) and treats ambient_sum as a plain sum
    loss = (fw * gws.double()).sum() + (fa * gas.double()).sum() + (fi * gim.double()).sum()
    loss.backward()
    gs, gr, ga = oracle_ops.composite_rays_train_backward(gws, gas, gim, sig, rgb, amb, deltas, rays, ws, asum, image, T_thresh)
    assert (gr.double() - rd_.grad).abs().max().item() < 2e-5
    assert (ga.double() - ad.grad).abs().max().item() < 1e-6
    if T_thresh < 1e-3:
        # with (almost) no cut the closed form d/dsigma = dt * (g_img . (T c - (C_final - C_k)) + g_ws (1 - ws_final)) is the exact gradient
        assert (gs.double() - sd.grad).abs().max().item() < 5e-4 * max(1.0, sd.grad.abs().max().item())
    else:
        # after an early break the formula still uses the FINAL sums, i.e. it is the gradient of the truncated integral: same check
        assert (gs.double() - sd.grad).abs().max().item() < 5e-4 * max(1.0, sd.grad.abs().max().item())


def test_march_train_backward_is_the_adjoint_of_the_sample_positions(oracle_ops):
    sc, ro, rd, nears, fars = _rays(oracle_ops, H=24)
    xyzs, dirs, deltas, rays, counter = oracle_ops.march_rays_train(ro, rd, 1.0, sc.state["density_bitfield"], 1, 128, nears, fars, dt_gamma=1 / 256, max_steps=16)
    M = int(counter[0])
    g = torch.Generator().manual_seed(1)
    gx, gd = torch.randn(xyzs.shape[0], 3, generator=g), torch.randn(xyzs.shape[0], 3, generator=g)
    go, gdd = oracle_ops.march_rays_train_backward(gx, gd, rays, deltas)
    n = int(torch.argmax(rays[:, 2]))
    o, k = int(rays[n, 1]), int(rays[n, 2])
    assert k > 3 and o + k <= M
    assert torch.allclose(go[n], gx[o:o + k].sum(0), atol=1e-5)
    assert torch.allclose(gdd[n], (gx[o:o + k] * deltas[o:o + k, 1:2]).sum(0) + gd[o:o + k].sum(0), atol=1e-4)


@pytest.mark.parametrize("D,gridtype,interp", [(3, 1, 0), (2, 1, 0), (3, 0, 1)])
def test_grid_backward_is_the_adjoint_of_the_forward_and_dydx_matches_finite_differences(oracle_ops, D, gridtype, interp):
    lay = GridLayout(D, log2_hashmap_size=14 if gridtype == 0 else 16, desired_resolution=512, gridtype="hash" if gridtype == 0 else "tiled")
    offsets = torch.from_numpy(np.asarray(lay.offsets, dtype=np.int32))
    n_entries = int(offsets[-1])
    g = torch.Generator().manual_seed(D * 10 + gridtype)
    table = torch.rand(n_entries, 2, generator=g) - 0.5
    B = 300
    x = torch.rand(B, D, generator=g) * 0.98 + 0.01
    x[5] = 1.5                                                                                              # out of range: no contribution
    G = torch.randn(B, 32, generator=g)
    y = oracle_ops.grid_encode(x, table, offsets, lay.per_level_scale, 16, gridtype, False, interp)
    dydx = oracle_ops.grid_encode_dydx(x, table, offsets, lay.per_level_scale, 16, gridtype, False, interp)
    ge, gi = oracle_ops.grid_encode_backward(G, x, table, offsets, lay.per_level_scale, 16, gridtype, False, interp, dy_dx=dydx)
    # forward is linear in the table: <forward(T), G> == <T, backward(G)>
    lhs, rhs = (y.double() * G.double()).sum().item(), (table.double() * ge.double()).sum().item()
    assert abs(lhs - rhs) < 1e-3 * max(1.0, abs(lhs))
    assert gi[5].abs().sum().item() == 0 and dydx[5].abs().sum().item() == 0
    # input gradient against central differences of the forward (coarse levels only: fine cells are narrower than the step)
    h = 1e-4
    for d in range(D):
        e = torch.zeros(B, D); e[:, d] = h
        num = (oracle_ops.grid_encode(x + e, table, offsets, lay.per_level_scale, 16, gridtype, False, interp) -
               oracle_ops.grid_encode(x - e, table, offsets, lay.per_level_scale, 16, gridtype, False, interp)) / (2 * h)          # [B, 32]
        ana = dydx[:, :, d, :].reshape(B, 32)
        ok = torch.ones(B, dtype=torch.bool); ok[5] = False
        err = (num[ok, :8] - ana[ok, :8]).abs()
        assert err.median().item() < 2e-2 * max(1.0, ana[ok, :8].abs().max().item())
    # the same adjoint identity for the input gradient: grad_inputs[b,d] = sum_{l,c} G[b,l,c] dy_dx[b,l,d,c]
    ref = torch.einsum("blc,bldc->bd", G.view(B, 16, 2).double(), dydx.double())
    assert (gi.double() - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())


def test_morton_packbits_dilation_identities(oracle_ops):
    g = torch.Generator().manual_seed(3)
    coords = torch.randint(0, 128, (500, 3), generator=g, dtype=torch.int32)
    idx = oracle_ops.morton3D(coords)
    assert torch.equal(oracle_ops.morton3D_invert(idx), coords)
    H = 16
    dense = torch.rand(H, H, H, generator=g)
    xs = torch.stack(torch.meshgrid(torch.arange(H), torch.arange(H), torch.arange(H), indexing="ij"), -1).view(-1, 3).int()
    mi = oracle_ops.morton3D(xs).long()
    grid = torch.zeros(1, H ** 3); grid[0, mi] = dense.view(-1)
    dil = oracle_ops.morton3D_dilation(grid)
    p = torch.nn.functional.pad(dense[None, None], (1, 1, 1, 1, 1, 1), value=-1.0)[0, 0]
    ref = dense.clone()
    for sh in ((0, 1, 1), (2, 1, 1), (1, 0, 1), (1, 2, 1), (1, 1, 0), (1, 1, 2)):
        ref = torch.maximum(ref, p[sh[0]:sh[0] + H, sh[1]:sh[1] + H, sh[2]:sh[2] + H])
    assert torch.equal(dil[0, mi], ref.view(-1))
    bits = oracle_ops.packbits(grid, 0.5)
    assert np.array_equal(bits.numpy(), np.packbits((grid.view(-1).numpy() > 0.5).astype(np.uint8), bitorder="little"))
    ro = torch.randn(50, 3, generator=g) * 0.3
    rd = torch.nn.functional.normalize(torch.randn(50, 3, generator=g), dim=-1)
    c = oracle_ops.sph_from_ray(ro, rd, 2.0)
    theta, phi = (c[:, 0] + 1) * np.pi / 2, c[:, 1] * np.pi
    p_ = 2.0 * torch.stack([torch.sin(theta) * torch.cos(phi), torch.cos(theta), torch.sin(theta) * torch.sin(phi)], -1)     # y up
    t = ((p_ - ro) * rd).sum(-1, keepdim=True)
    assert (ro + t * rd - p_).abs().max().item() < 1e-4 and (t > 0).all()
