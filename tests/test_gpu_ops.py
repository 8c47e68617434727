"""Per-op parity on the GPU: every (A)-level entry point of the C-ABI vs the C oracle on the same inputs.

Integer / discrete results (near/far, marched positions, which rows are written, alive flags) must be
bit-exact; smooth fp32 results within 2e-6 relative (different FMA contraction only)."""
import ctypes

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import _capi, scene as scn
from genefaceplusplus_b200.config import GridLayout

pytestmark = pytest.mark.gpu


_KEEP = []


def P(t):
    """Device pointer; the tensor is kept alive until the end of the test module (P(x.cuda()) would otherwise hand
    the kernel a pointer the caching allocator has already recycled)."""
    _KEEP.append(t)
    return ctypes.c_void_p(t.data_ptr())


def S():
    return _capi.stream_ptr()


@pytest.fixture(scope="module")
def rays():
    sc = scn.Scene(H=96, W=96, T=4, torso=False)
    fi = sc.frame_inputs(1)
    return sc, fi["rays_o"].view(-1, 3).contiguous(), fi["rays_d"].view(-1, 3).contiguous()


def test_device_is_hopper():
    _capi.check(_capi.lib().gfpp_check_device(), "check_device")


def test_near_far_bit_exact(rays, oracle_ops):
    sc, ro, rd = rays
    aabb = sc.state["aabb_infer"]
    n_ref, f_ref = oracle_ops.near_far_from_aabb(ro, rd, aabb, 0.05)
    N = ro.shape[0]
    nears = torch.empty(N, device="cuda"); fars = torch.empty(N, device="cuda")
    _capi.check(_capi.lib().gfpp_near_far_from_aabb(P(ro.cuda()), P(rd.cuda()), P(aabb.cuda()), N, 0.05, P(nears), P(fars), S()))
    assert torch.equal(nears.cpu(), n_ref) and torch.equal(fars.cpu(), f_ref)
    # rays that miss the box: both FLT_MAX
    ro2 = ro.clone(); ro2[:, 1] += 5.0
    n2, f2 = oracle_ops.near_far_from_aabb(ro2, rd, aabb, 0.05)
    _capi.check(_capi.lib().gfpp_near_far_from_aabb(P(ro2.cuda()), P(rd.cuda()), P(aabb.cuda()), N, 0.05, P(nears), P(fars), S()))
    assert torch.equal(nears.cpu(), n2) and torch.equal(fars.cpu(), f2)
    assert (n2 == torch.finfo(torch.float32).max).any()


@pytest.mark.parametrize("n_step,max_steps,dt_gamma", [(1, 16, 1 / 256), (4, 16, 1 / 256), (8, 1024, 1 / 256), (3, 64, 0.0)])
def test_march_rays_bit_exact(rays, oracle_ops, n_step, max_steps, dt_gamma):
    sc, ro, rd = rays
    aabb = sc.state["aabb_infer"]
    bits = sc.state["density_bitfield"]
    nears, fars = oracle_ops.near_far_from_aabb(ro, rd, aabb, 0.05)
    N = ro.shape[0]
    alive = torch.arange(N, dtype=torch.int32)[::2].contiguous()  # ragged subset
    n_alive = alive.shape[0]
    rays_t = nears.clone()
    for rnd in range(3):  # several rounds so that later rounds start mid-volume
        x_ref, d_ref, l_ref = oracle_ops.march_rays(n_alive, n_step, alive, rays_t, ro, rd, 1.0, bits, 1, 128, nears, fars, 128, False, dt_gamma, max_steps)
        M = x_ref.shape[0]
        xyzs = torch.zeros(M, 3, device="cuda"); dirs = torch.zeros(M, 3, device="cuda"); deltas = torch.zeros(M, 2, device="cuda")
        noises = torch.zeros(n_alive, device="cuda")
        _capi.check(_capi.lib().gfpp_march_rays(n_alive, n_step, P(alive.cuda()), P(rays_t.cuda()), P(ro.cuda()), P(rd.cuda()), 1.0, dt_gamma,
                                                max_steps, 1, 128, P(bits.cuda()), P(nears.cuda()), P(fars.cuda()), P(xyzs), P(dirs), P(deltas), P(noises), S()))
        assert torch.equal(xyzs.cpu(), x_ref), f"round {rnd}: positions differ"
        assert torch.equal(deltas.cpu(), l_ref), f"round {rnd}: deltas differ"
        assert torch.equal(dirs.cpu(), d_ref)
        assert (l_ref[:, 0] > 0).sum() > 100  # the case is not vacuous
        # advance like the compositor would (t = last delta[1] of rays that used all their steps)
        last = l_ref[: n_alive * n_step].view(n_alive, n_step, 2)[:, -1, :]
        full = last[:, 0] > 0
        rays_t[alive[full].long()] = last[full, 1]


def test_composite_rays(oracle_ops):
    g = torch.Generator().manual_seed(3)
    N, n_alive, n_step = 500, 300, 4
    alive = torch.randperm(N, generator=g)[:n_alive].int().contiguous()
    M = n_alive * n_step + 128 - (n_alive * n_step) % 128
    sig = torch.rand(M, generator=g) * 40
    rgb = torch.rand(M, 3, generator=g)
    deltas = torch.zeros(M, 2)
    deltas[: n_alive * n_step, 0] = 0.027
    deltas[: n_alive * n_step, 1] = torch.rand(n_alive * n_step, generator=g) + 3
    # some rays run out early (delta == 0 rows)
    dl = deltas[: n_alive * n_step].view(n_alive, n_step, 2)
    dl[::7, 2:, :] = 0
    ws = torch.rand(N, generator=g) * 0.9; dp = torch.rand(N, generator=g); img = torch.rand(N, 3, generator=g); t = torch.rand(N, generator=g)
    ref = [x.clone() for x in (alive, t, ws, dp, img)]
    oracle_ops.composite_rays(n_alive, n_step, ref[0], ref[1], sig, rgb, deltas, ref[2], ref[3], ref[4], 0.05)
    dev = [x.clone().cuda() for x in (alive, t, ws, dp, img)]
    _capi.check(_capi.lib().gfpp_composite_rays(n_alive, n_step, 0.05, P(dev[0]), P(dev[1]), P(sig.cuda()), P(rgb.cuda()), P(deltas.cuda()), P(dev[2]), P(dev[3]), P(dev[4]), S()))
    assert torch.equal(dev[0].cpu(), ref[0])          # which rays die: exact
    assert torch.equal(dev[1].cpu(), ref[1])          # rays_t: exact (copied values)
    for a, b in zip(dev[2:], ref[2:]):
        assert (a.cpu() - b).abs().max().item() < 2e-6
    assert (ref[0] < 0).sum() > 10 and (ref[0] >= 0).sum() > 10


@pytest.mark.parametrize("D,gridtype,interp", [(3, "tiled", "linear"), (2, "tiled", "linear"), (3, "hash", "linear"), (3, "tiled", "smoothstep"), (2, "hash", "smoothstep")])
def test_grid_encode(oracle_ops, D, gridtype, interp):
    lay = GridLayout(D, gridtype=gridtype, interpolation=interp)
    g = torch.Generator().manual_seed(D)
    emb = (torch.rand(lay.n_entries, 2, generator=g) - 0.5)
    B = 5000
    x = torch.rand(B, D, generator=g)
    x[:7] = 0.0; x[7:14] = 1.0          # the closed ends of [0,1]
    x[14] = -0.01; x[15] = 1.01         # out of range => zeros (gridencoder.cu:110-135)
    off = torch.from_numpy(lay.offsets.copy())
    ref = oracle_ops.grid_encode(x, emb, off, lay.per_level_scale, 16, lay.gridtype_id, False, lay.interp_id)
    out = torch.empty(16, B, 2, device="cuda")
    offs = np.ascontiguousarray(lay.offsets)
    _capi.check(_capi.lib().gfpp_grid_encode_forward(P(x.cuda()), P(emb.cuda()), offs.ctypes.data, P(out), B, D, 2, 16, float(lay.S), 16,
                                                     lay.gridtype_id, 0, lay.interp_id, S()))
    mine = out.permute(1, 0, 2).reshape(B, 32).cpu()
    assert (mine[14:16] == 0).all()
    assert (mine - ref).abs().max().item() < 2e-6


def test_grid_encode_rejects_unsupported_shapes():
    L = _capi.lib()
    x = torch.zeros(4, 3, device="cuda")
    off = np.zeros(17, dtype=np.int32)
    assert L.gfpp_grid_encode_forward(P(x), P(x), off.ctypes.data, P(x), 4, 3, 4, 16, 0.46, 16, 1, 0, 0, S()) == -4   # C=4
    assert L.gfpp_grid_encode_forward(P(x), P(x), off.ctypes.data, P(x), 4, 5, 2, 16, 0.46, 16, 1, 0, 0, S()) == -4   # D=5


@pytest.mark.parametrize("degree", [1, 2, 3, 4])
def test_sh_encode(oracle_ops, degree):
    g = torch.Generator().manual_seed(0)
    d = torch.nn.functional.normalize(torch.randn(4097, 3, generator=g), dim=-1)
    ref = oracle_ops.sh_encode(d, degree)
    out = torch.empty(4097, degree * degree, device="cuda")
    _capi.check(_capi.lib().gfpp_sh_encode_forward(P(d.cuda()), P(out), 4097, 3, degree, S()))
    assert (out.cpu() - ref).abs().max().item() < 1e-6


@pytest.mark.parametrize("D,deg", [(2, 10), (6, 4)])
def test_freq_encode(oracle_ops, D, deg):
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(3001, D, generator=g) * 2 - 1) * (0.8 if D == 2 else 4.0)
    ref = oracle_ops.freq_encode(x, deg)
    C = D + 2 * D * deg
    out = torch.empty(3001, C, device="cuda")
    _capi.check(_capi.lib().gfpp_freq_encode_forward(P(x.cuda()), 3001, D, deg, C, P(out), S()))
    # accurate sinf on arguments up to 2^9 * 0.8 rad (the reference's __sinf would be off by >> 1e-3 there)
    assert (out.cpu() - ref).abs().max().item() < 2e-6


def test_empty_inputs_are_noops():
    L = _capi.lib()
    z = torch.zeros(1, device="cuda")
    assert L.gfpp_near_far_from_aabb(P(z), P(z), P(z), 0, 0.05, P(z), P(z), S()) == 0
    assert L.gfpp_sh_encode_forward(P(z), P(z), 0, 3, 4, S()) == 0
    torch.cuda.synchronize()
