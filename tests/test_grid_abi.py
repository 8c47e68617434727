"""C-ABI section (E), occupancy-grid maintenance: argument validation happens before any CUDA call, so it is checked without a
GPU; a model on the CPU raises instead of falling back."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso

P = ctypes.c_void_p


def test_workspace_query_and_shapes():
    L = _capi.lib()
    assert L.gfpp_density_grid_workspace_bytes(1, 128) >= 128 ** 3 * 4
    assert L.gfpp_density_grid_workspace_bytes(1, 32) >= 32 ** 3 * 4
    for C, H in ((0, 128), (9, 128), (1, 6), (1, 130), (1, 96), (1, 1024)):
        assert L.gfpp_density_grid_workspace_bytes(C, H) == 0, (C, H)


def test_entry_points_validate_before_any_cuda_call():
    L = _capi.lib()
    m = _capi.Model()                                                   # never packed
    assert L.gfpp_density_query(None, P(16), 4, P(16), P(16), None, None) == -1 and b"null" in L.gfpp_last_error()
    assert L.gfpp_density_query(ctypes.byref(m), P(16), 4, P(16), P(16), None, None) == -1
    assert b"gfpp_model_pack" in L.gfpp_last_error()
    assert L.gfpp_density_grid_update(ctypes.byref(m), P(16), P(16), 0.95, 10.0, P(16), P(16), None, P(16), 1 << 30, None) == -1
    assert b"gfpp_model_pack" in L.gfpp_last_error()
    assert L.gfpp_density_grid_update(ctypes.byref(m), None, P(16), 0.95, 10.0, P(16), P(16), None, P(16), 1 << 30, None) == -1
    assert b"null" in L.gfpp_last_error()
    assert L.gfpp_mark_untrained_grid(None, 1, 1.0, 1.0, 0.5, 0.5, 1.0, 1, 128, P(16), None) == -1
    assert L.gfpp_mark_untrained_grid(P(16), 1, 1.0, 1.0, 0.5, 0.5, 1.0, 9, 128, P(16), None) == -4     # cascade
    assert L.gfpp_mark_untrained_grid(P(16), 1, 1.0, 1.0, 0.5, 0.5, 1.0, 1, 100 + 2, P(16), None) == -4  # grid_size
    assert L.gfpp_mark_untrained_grid(P(16), 0, 1.0, 1.0, 0.5, 0.5, 1.0, 1, 128, P(16), None) == -1      # no poses


def test_handle_without_a_grid_shape_is_unsupported():
    """A handle that carries the pack's magic but cascade = grid_size = 0 is refused before any launch (the short-workspace
    check needs a really packed model: tests/test_gpu_grid.py)."""
    L = _capi.lib()
    m = _capi.Model()
    m.opaque[0] = 0x67667070                      # the magic gfpp_model_pack writes first ("gfpp")
    assert L.gfpp_density_grid_update(ctypes.byref(m), P(16), P(16), 0.95, 10.0, P(16), P(16), None, P(16), 1 << 30, None) == -4
    assert b"grid_size" in L.gfpp_last_error()


def test_cpu_model_raises():
    hp = may_hparams(grid_size=32)
    model = RADNeRF(hp)
    model.load_state_dict(scn.make_state(torso=False, hparams=hp), strict=True)
    model.conds = scn.cond_sequence(4)
    with pytest.raises(_capi.GfppError):
        model.update_extra_state(cond_index=1)
    with pytest.raises(_capi.GfppError):
        model.density(torch.zeros(4, 3), torch.zeros(64))
    with pytest.raises(_capi.GfppError):
        model.mark_untrained_grid(torch.eye(4).unsqueeze(0), (100.0, 100.0, 16.0, 16.0))
    torso = RADNeRFTorso(may_hparams())
    with pytest.raises(NotImplementedError):
        torso.update_extra_state()


@pytest.mark.parametrize("S", [128, 16, 12])
def test_cell_noise_follows_the_reference_draw_order(S):
    """update_extra_state's default jitter: the reference draws rand_like([n, 3]) per chunk of cells (x-, then y-, then z-chunks of S,
    renderer.py:234-258) and per cascade inside each chunk; the [C,H,H,H,3] tensor must hold those draws at their cells."""
    hp = may_hparams(grid_size=32, bound=2)
    model = RADNeRF(hp)
    H, C = model.grid_size, model.cascade
    assert C == 2
    torch.manual_seed(7)
    got = model._cell_noise(S, torch.device("cpu"))
    torch.manual_seed(7)
    want = torch.empty(C, H, H, H, 3)
    r = torch.arange(H, dtype=torch.int32)
    for xs in r.split(S):
        for ys in r.split(S):
            for zs in r.split(S):
                xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing="ij")
                coords = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1).long()
                for cas in range(C):
                    want[cas, coords[:, 0], coords[:, 1], coords[:, 2]] = torch.rand_like(coords.float())
    assert torch.equal(got, want)
