"""Occupancy-grid maintenance on the GPU (k_density in head_kernel.cu, grid_kernels.cu, gfpp.h section E) against the reference's own
update_extra_state / mark_untrained_grid outputs (tests/golden/grid_*.npz) and the CPU oracle (oracle/grid.py).

The density query evaluates the field the model's mode renders: fp16 models run k_density_tc (fp16 operands and oct tables on wgmma,
what the reference computes under autocast); fp32, bf16x3, bf16 and robust models run the fp32 FFMA field (the tests check that robust
gives the fp32 result bit for bit).  Bitfield cells may flip only when their EMA value lies within the mode's band (relative) of the
threshold: the GPU sums in another order than the CPU (fp32), or rounds operands to fp16.  The fp16 bounds are about twice the errors
the first H100 run measured (raw 4.3e-4, geo_feat 8.9e-4, mean 3.4e-7; 5 of 2 097 152 cells flipped at 128^3).  Flip counts and errors are printed."""
import ctypes
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.renderer import RADNeRF
from oracle import grid as og
from oracle import make_grid_golden as mg
from oracle.render import OracleModel

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# per mode: raw density (relative), geo_feat (absolute), mean (relative), band around the threshold within which a cell may flip
BOUNDS = {"fp32": dict(raw=2e-5, geo=1e-5, mean=1e-5, band=1e-4), "fp16": dict(raw=1e-3, geo=2e-3, mean=1e-6, band=1e-3)}


def _golden(name):
    return np.load(os.path.join(GOLDEN, name))


def _model(H, precision="fp32"):
    inp = mg.inputs(H)
    m = RADNeRF(inp["hp"])
    m.load_state_dict(inp["state"], strict=True)
    m.density_scale = mg.DS
    m.mlp_precision = precision
    m.conds = inp["conds"]
    return m.cuda().eval(), inp


def _bit_flips(bits_gpu, bits_ref, ema_gpu, thr, band):
    """(flipped cells, flipped cells outside the band)."""
    a = np.unpackbits(bits_gpu, bitorder="little")
    b = np.unpackbits(bits_ref, bitorder="little")
    flip = a != b
    near = np.abs(ema_gpu.reshape(-1) - thr) <= band * thr
    return int(flip.sum()), int((flip & ~near).sum())


@pytest.mark.parametrize("precision", ["fp32", "fp16", "robust"])
def test_density_query_vs_oracle(oracle_ops, precision):
    m, inp = _model(32, precision)
    g = _golden("grid_head32.npz")
    cf = torch.from_numpy(g["cond_feat"])
    x = scn.hashed_uniform(3 * 65536, 17, 2.0).view(-1, 3)
    out = m.density(x.cuda(), cf.cuda())
    torch.cuda.synchronize()
    orc = OracleModel(inp["state"], inp["hp"], torso=False)
    sig, geo = og.density(orc, x, cf)
    ds = ((out["sigma"].cpu() - sig).abs() / sig.abs()).max().item()
    dg = (out["geo_feat"].cpu() - geo).abs().max().item()
    print(f"[density {precision}] 65536 points: max rel |sigma - fp32 oracle| {ds:.3e}, max |geo_feat - fp32 oracle| {dg:.3e}")
    b = BOUNDS["fp16" if precision == "fp16" else "fp32"]
    assert ds <= b["raw"] and dg <= b["geo"]
    if precision == "robust":     # robust renders a split-precision approximation of the fp32 field: its grid comes from that field
        ref, _ = _model(32, "fp32")
        o32 = ref.density(x.cuda(), cf.cuda())
        assert torch.equal(o32["sigma"], out["sigma"]) and torch.equal(o32["geo_feat"], out["geo_feat"])


@pytest.mark.parametrize("H,precision", [(32, "fp32"), (32, "fp16"), (128, "fp32"), (128, "fp16")])
def test_refresh_vs_reference(H, precision):
    g = _golden(f"grid_head{H}.npz")
    m, inp = _model(H, precision)
    C = m.cascade
    tmp = torch.empty(C, H ** 3, device="cuda")
    mean = m.refresh_density_grid(torch.from_numpy(g["cond_feat"]), inp["noise"], mg.DECAY, tmp_grid=tmp)
    torch.cuda.synchronize()
    raw, ema = tmp.cpu().reshape(-1), m.density_grid.cpu().reshape(-1)
    idx = torch.arange(raw.numel()) if H == 32 else torch.from_numpy(g["cells"])
    graw, gema = torch.from_numpy(g["raw"]).reshape(-1), torch.from_numpy(g["ema"]).reshape(-1)
    d_raw = ((raw[idx] - graw).abs() / graw.abs().clamp(min=1)).max().item()
    d_ema = ((ema[idx] - gema).abs() / gema.abs().clamp(min=1)).max().item()
    gm = float(g["mean"][0])
    d_mean = abs(mean.item() - gm) / gm
    thr = min(gm, float(inp["hp"]["density_thresh"]))
    b = BOUNDS[precision]
    n_flip, n_bad = _bit_flips(m.density_bitfield.cpu().numpy(), g["bitfield"], ema.numpy(), thr, b["band"])
    occ = np.unpackbits(m.density_bitfield.cpu().numpy()).mean()
    print(f"[refresh {H}^3 {precision}] rel err raw {d_raw:.3e}, EMA {d_ema:.3e}, mean {d_mean:.3e}; bitfield flips {n_flip} "
          f"of {8 * g['bitfield'].size} cells (outside the {b['band']:g} band: {n_bad}); occupancy {occ:.3f}")
    assert d_raw <= b["raw"] and d_ema <= b["raw"] and d_mean <= b["mean"] and n_bad == 0
    assert 0.05 < occ < 0.95
    untrained = inp["grid0"].reshape(-1) == -1
    assert bool((ema[untrained] == -1).all())


def test_refresh_is_deterministic():
    g = _golden("grid_head128.npz")
    outs = []
    for _ in range(2):
        m, inp = _model(128, "fp16")
        mean = m.refresh_density_grid(torch.from_numpy(g["cond_feat"]), inp["noise"], mg.DECAY)
        outs.append((m.density_grid.clone(), mean.clone(), m.density_bitfield.clone()))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))


def test_short_workspace_is_refused():
    m, inp = _model(32)
    _, _, model, _ = m._ensure_packed()
    L = _capi.lib()
    need = L.gfpp_density_grid_workspace_bytes(1, 32)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    cf = torch.zeros(64, device="cuda")
    noise = inp["noise"].cuda()
    mean = torch.empty(1, device="cuda")
    rc = L.gfpp_density_grid_update(ctypes.byref(model), cf.data_ptr(), noise.data_ptr(), 0.95, 10.0, m.density_grid.data_ptr(),
                                    mean.data_ptr(), None, ws.data_ptr(), need - 1, _capi.stream_ptr())
    assert rc == -3 and b"workspace" in L.gfpp_last_error()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_render_after_update_matches_a_fresh_model(precision):
    """update_extra_state rewrites the bitfield and the packed occupancy in place; the next render_clip must be the one a model
    packed from the updated state renders, bit for bit."""
    sc = scn.Scene(H=64, W=64, T=2, torso=False, density_scale=mg.DS)
    m = RADNeRF(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale, m.mlp_precision, m.conds = sc.density_scale, precision, sc.cond
    m = m.cuda().eval()
    poses = torch.stack([sc.pose(t) for t in range(2)]).cuda()
    before = m.render_clip(poses, sc.intrinsics, 64, 64, cond_seq=sc.cond.cuda(), T_thresh=sc.T_thresh)
    packed_before = m._packed[1]
    noise = (scn.hashed_uniform(128 ** 3 * 3, 7, 1.0) + 0.5).view(1, 128, 128, 128, 3)
    m.update_extra_state(cond_index=1, noise=noise)
    after = m.render_clip(poses, sc.intrinsics, 64, 64, cond_seq=sc.cond.cuda(), T_thresh=sc.T_thresh)
    assert m._packed[1] is packed_before                      # not repacked
    fresh = RADNeRF(sc.hparams)
    fresh.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    fresh.density_scale, fresh.mlp_precision = sc.density_scale, precision
    fresh = fresh.cuda().eval()
    ref = fresh.render_clip(poses, sc.intrinsics, 64, 64, cond_seq=sc.cond.cuda(), T_thresh=sc.T_thresh)
    torch.cuda.synchronize()
    changed = (after != before).any().item()
    print(f"[render after update, {precision}] mean_density {m.mean_density:.4f}; frames changed by the refresh: {changed}; "
          f"max|after - fresh model| {(after - ref).abs().max().item():.3e}")
    assert torch.equal(after, ref)


def test_mark_untrained_vs_reference():
    g = _golden("grid_untrained128.npz")
    m, _ = _model(128)
    m.density_grid.zero_()
    poses, intr = mg.untrained_inputs()
    m.mark_untrained_grid(poses, intr)
    torch.cuda.synchronize()
    mine = np.packbits((m.density_grid.cpu().reshape(-1) == -1).numpy().astype(np.uint8))
    flips = int(np.unpackbits(mine ^ g["untrained_bits"]).sum())
    print(f"[mark_untrained_grid] {int(g['n_untrained'][0])} untrained cells in the reference; cells that differ: {flips}")
    assert flips == 0


def test_refresh_two_cascades_vs_oracle(oracle_ops, monkeypatch):
    """bound 2 => two cascades: per-cascade cell scale / jitter and the cascade offset of the noise and grid indices."""
    from genefaceplusplus_b200.config import may_hparams
    H = 32
    hp = may_hparams(grid_size=H, bound=2)
    monkeypatch.setattr(scn, "cascade_count", lambda b: 1)         # make_state builds cascade-0 occupancy only
    state = scn.make_state(torso=False, hparams=hp)
    monkeypatch.undo()
    C = 2
    grid0 = (scn.hashed_uniform(C * H ** 3, 412, 1.0) + 0.5).reshape(C, -1) * (2 * mg.DS)
    grid0.view(-1)[::5] = -1.0
    state["density_grid"] = grid0.clone()
    state["density_bitfield"] = torch.zeros(C * H ** 3 // 8, dtype=torch.uint8)
    noise = (scn.hashed_uniform(C * H ** 3 * 3, 411, 1.0) + 0.5).reshape(C, H, H, H, 3)
    m = RADNeRF(hp)
    assert m.cascade == C
    m.load_state_dict(state, strict=True)
    m.density_scale = mg.DS
    m = m.cuda().eval()
    cf = torch.from_numpy(_golden("grid_head32.npz")["cond_feat"])
    tmp = torch.empty(C, H ** 3, device="cuda")
    mean = m.refresh_density_grid(cf, noise, mg.DECAY, tmp_grid=tmp)
    torch.cuda.synchronize()
    orc = OracleModel(state, hp, torso=False)
    orc.density_scale = mg.DS
    assert orc.cascade == C
    o_tmp, o_grid, o_mean, o_bits = og.update_extra_state(orc, cf, noise, grid0, mg.DECAY, float(hp["density_thresh"]))
    d_raw = ((tmp.cpu() - o_tmp).abs() / o_tmp.abs().clamp(min=1)).max().item()
    d_ema = ((m.density_grid.cpu() - o_grid).abs() / o_grid.abs().clamp(min=1)).max().item()
    d_mean = abs(mean.item() - o_mean) / o_mean
    thr = min(o_mean, float(hp["density_thresh"]))
    b = BOUNDS["fp32"]
    n_flip, n_bad = _bit_flips(m.density_bitfield.cpu().numpy(), o_bits.numpy(), m.density_grid.cpu().numpy(), thr, b["band"])
    print(f"[refresh 2 cascades {H}^3] rel err raw {d_raw:.3e}, EMA {d_ema:.3e}, mean {d_mean:.3e}; bitfield flips {n_flip} (outside the band: {n_bad})")
    assert d_raw <= b["raw"] and d_ema <= b["raw"] and d_mean <= b["mean"] and n_bad == 0
