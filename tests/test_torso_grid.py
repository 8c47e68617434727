"""The torso occupancy-grid refresh without a GPU: C-ABI section (F) validates its arguments before any CUDA call, the default jitter
follows the reference's draw order, the CPU oracle (oracle/torso_grid.py) reproduces the reference's own update_extra_state
(tests/golden/torso_*grid*.npz), and models on the CPU raise instead of falling back."""
import ctypes
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR
from oracle import make_torso_grid_golden as mtg
from oracle import torso_grid as otg
from oracle.render import OracleModel

P = ctypes.c_void_p
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODEL_MAGIC, TORSO_SR_MAGIC = 0x67667070, 0x67667473     # what gfpp_model_pack / gfpp_torso_sr_pack write first


def test_workspace_query():
    L = _capi.lib()
    assert L.gfpp_torso_grid_workspace_bytes(128) >= 128 * 128 * 4 + 96 * 4
    assert L.gfpp_torso_grid_workspace_bytes(2) > 0 and L.gfpp_torso_grid_workspace_bytes(4096) > 0
    q = L.gfpp_torso_query_workspace_bytes()
    assert 96 * 4 <= q <= L.gfpp_torso_grid_workspace_bytes(2)          # the folded biases; a refresh workspace serves the query too
    for H in (0, 1, 4097):
        assert L.gfpp_torso_grid_workspace_bytes(H) == 0, H


def _update(L, m, code=None, ws_bytes=1 << 30, grid=P(16)):
    return L.gfpp_torso_grid_update(ctypes.byref(m), P(16), code, P(16), 0.95, grid, P(16), None, P(16), ws_bytes, None)


def test_entry_points_validate_before_any_cuda_call():
    L = _capi.lib()
    m = _capi.Model()                                                   # never packed
    assert L.gfpp_torso_query(None, P(16), 4, P(16), None, P(16), None, None, P(16), 1 << 20, None) == -1
    assert b"null" in L.gfpp_last_error()
    assert L.gfpp_torso_query(ctypes.byref(m), P(16), 4, P(16), None, P(16), None, None, P(16), 1 << 20, None) == -1
    assert b"gfpp_model_pack" in L.gfpp_last_error()
    assert _update(L, m) == -1 and b"gfpp_model_pack" in L.gfpp_last_error()
    assert _update(L, m, grid=None) == -1 and b"null" in L.gfpp_last_error()
    m.opaque[0] = MODEL_MAGIC                                           # packed, but without a torso (has_torso = 0)
    assert _update(L, m) == -1 and b"has_torso" in L.gfpp_last_error()
    assert L.gfpp_torso_query(ctypes.byref(m), P(16), 4, P(16), None, P(16), None, None, P(16), 1 << 20, None) == -1
    assert b"has_torso" in L.gfpp_last_error()
    assert L.gfpp_model_set_torso_threshold(ctypes.byref(m), 0.01) == -1 and b"has_torso" in L.gfpp_last_error()
    m.opaque[0] = MODEL_MAGIC | (1 << 32)                               # has_torso = 1, torso_code_dim = 0, grid_size = 0
    assert _update(L, m, code=P(16)) == -1 and b"code" in L.gfpp_last_error()
    assert _update(L, m) == -4 and b"grid_size" in L.gfpp_last_error()
    q = L.gfpp_torso_query_workspace_bytes()
    assert L.gfpp_torso_query(ctypes.byref(m), P(16), 4, P(16), None, P(16), None, None, P(16), q - 1, None) == -3
    assert b"workspace" in L.gfpp_last_error()
    assert L.gfpp_model_set_torso_threshold(None, 0.01) == -1
    sm = _capi.TorsoSrModel()
    args = (P(16), None, P(16), 0.95, P(16), P(16), None, P(16), 1 << 30, None)
    assert L.gfpp_torso_sr_grid_update(ctypes.byref(sm), *args) == -1 and b"gfpp_torso_sr_pack" in L.gfpp_last_error()
    assert L.gfpp_torso_sr_grid_update(None, *args) == -1 and b"null" in L.gfpp_last_error()
    assert L.gfpp_torso_sr_set_threshold(ctypes.byref(sm), 0.01) == -1 and b"gfpp_torso_sr_pack" in L.gfpp_last_error()
    sm.opaque[0] = TORSO_SR_MAGIC                                       # code_dim = 0, grid_size = 0
    assert L.gfpp_torso_sr_grid_update(ctypes.byref(sm), P(16), P(16), *args[2:]) == -1 and b"code" in L.gfpp_last_error()
    assert L.gfpp_torso_sr_grid_update(ctypes.byref(sm), *args) == -4 and b"grid_size" in L.gfpp_last_error()
    assert L.gfpp_torso_sr_set_threshold(ctypes.byref(sm), 0.01) == 0


@pytest.mark.parametrize("S", [128, 64, 48])
def test_torso_cell_noise_follows_the_reference_draw_order(S):
    """update_extra_state's default jitter: the reference draws rand_like([n, 2]) per chunk of cells (x-, then y-chunks of S,
    radnerf_torso.py:216-227); the [H,H,2] tensor must hold those draws at their cells."""
    model = RADNeRFTorso(may_hparams())
    H = model.grid_size
    assert H == 128
    torch.manual_seed(7)
    got = model._torso_cell_noise(S, torch.device("cpu"))
    torch.manual_seed(7)
    want = torch.empty(H, H, 2)
    r = torch.arange(H, dtype=torch.int32)
    for xs in r.split(S):
        for ys in r.split(S):
            xx, yy = torch.meshgrid(xs, ys, indexing="ij")
            coords = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1)], dim=-1).long()
            want[coords[:, 0], coords[:, 1]] = torch.rand_like(coords.float())
    assert torch.equal(got, want)


@pytest.mark.parametrize("name", list(mtg.CASES))
def test_oracle_reproduces_the_reference_refresh(oracle_ops, name):
    kind, H = mtg.CASES[name]
    g = np.load(os.path.join(GOLDEN, name))
    inp = mtg.inputs(kind, H)
    assert int(g["pose_index"][0]) == mtg.POSE_INDEX and np.array_equal(g["code"], inp["code"].numpy())
    orc = OracleModel(inp["state"], inp["hp"], torso=True)
    if kind == "torso_sr":
        assert np.array_equal(g["lm68"], inp["lm68s"][mtg.POSE_INDEX].numpy())
        kw = dict(lm68=torch.from_numpy(g["lm68"]))
    else:
        kw = dict(pose6=torch.from_numpy(g["pose6"]))
        # update_extra_state conditions on scene.convert_poses of the training pose: bit-equal to the reference's own conversion
        assert torch.equal(scn.convert_poses(inp["poses"][mtg.POSE_INDEX].view(1, 4, 4)).view(6), kw["pose6"])
    tmp, grid, mean = otg.update_extra_state(orc, inp["noise"], inp["grid0"], mtg.DECAY, code=inp["code"], **kw)
    d_raw = (tmp - torch.from_numpy(g["raw"])).abs().max().item()
    d_ema = (grid - torch.from_numpy(g["ema"])).abs().max().item()
    d_mean = abs(mean - float(g["mean"][0])) / float(g["mean"][0])
    assert d_raw <= 1e-7 and d_ema <= 1e-7 and d_mean <= 1e-7, (d_raw, d_ema, d_mean)
    # both sides of max(grid * decay, dilated alphas) are exercised
    won = (inp["grid0"] * mtg.DECAY >= torch.from_numpy(g["ema"])).float().mean().item()
    assert 0.2 < won < 0.8, won


def test_cpu_models_raise():
    torso = RADNeRFTorso(may_hparams(grid_size=32))
    torso.poses = torch.stack([scn.camera_pose(t) for t in range(4)])
    for call in (lambda: torso.update_extra_state(pose_index=1), lambda: torso.forward_torso(torch.zeros(4, 2), torch.zeros(1, 6)),
                 lambda: torso.refresh_torso_grid(torch.zeros(6), None, torch.zeros(32, 32, 2))):
        with pytest.raises(_capi.GfppNoCpuPath) as e:
            call()
        assert isinstance(e.value, NotImplementedError) and isinstance(e.value, _capi.GfppError)
    hp = may_hparams(grid_size=32, **mtg.SR_OVERRIDES)
    sr = RADNeRFTorsowithSR(hp)
    sr.poses, sr.lm68s = torso.poses, scn.lm68_sequence(4)
    with pytest.raises(_capi.GfppNoCpuPath):
        sr.update_extra_state(pose_index=1)


def test_code_row_is_checked_on_the_host():
    torso = RADNeRFTorso(may_hparams(grid_size=32))
    n = torso.torso_individual_codes.shape[0]
    assert torso._torso_code_row(n - 1, torch.device("cpu")).shape == (torso.torso_individual_embedding_dim,)
    for bad in (n, -1):
        with pytest.raises(IndexError):
            torso._torso_code_row(bad, torch.device("cpu"))
