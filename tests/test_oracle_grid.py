"""The CPU restatement of the occupancy-grid maintenance (oracle/grid.py) against the reference's own update_extra_state /
mark_untrained_grid outputs (tests/golden/grid_*.npz, written by oracle/make_grid_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import grid as og
from oracle import make_grid_golden as mg
from oracle.render import OracleModel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(name):
    return np.load(os.path.join(GOLDEN, name))


def _oracle(H):
    inp = mg.inputs(H)
    orc = OracleModel(inp["state"], inp["hp"], torso=False)
    orc.density_scale = mg.DS
    return orc, inp


@pytest.mark.parametrize("H", [32, 128])
def test_oracle_refresh_matches_reference(oracle_ops, H):
    g = _golden(f"grid_head{H}.npz")
    orc, inp = _oracle(H)
    tmp, grid, mean, bits = og.update_extra_state(orc, torch.from_numpy(g["cond_feat"]), inp["noise"], inp["grid0"], mg.DECAY,
                                                  float(inp["hp"]["density_thresh"]))
    if H == 32:
        assert torch.equal(tmp, torch.from_numpy(g["raw"])) and torch.equal(grid, torch.from_numpy(g["ema"]))
    else:
        idx = torch.from_numpy(g["cells"])
        assert torch.equal(tmp.reshape(-1)[idx], torch.from_numpy(g["raw"]))
        assert torch.equal(grid.reshape(-1)[idx], torch.from_numpy(g["ema"]))
    assert mean == float(g["mean"][0])
    assert torch.equal(bits, torch.from_numpy(g["bitfield"]))
    occ = np.unpackbits(g["bitfield"]).mean()
    assert 0.05 < occ < 0.95, occ                                      # the refreshed grid is neither empty nor full
    untrained = inp["grid0"] == -1
    assert bool((grid[untrained] == -1).all())                         # the EMA leaves untrained cells alone


def test_oracle_mark_untrained_matches_reference(oracle_ops):
    g = _golden("grid_untrained128.npz")
    orc, _ = _oracle(128)
    poses, intr = mg.untrained_inputs()
    out = og.mark_untrained_grid(orc, torch.zeros(1, 128 ** 3), poses, intr)
    bits = np.packbits((out.reshape(-1) == -1).numpy().astype(np.uint8))
    assert np.array_equal(bits, g["untrained_bits"])
    assert 0 < int(g["n_untrained"][0]) < 128 ** 3
