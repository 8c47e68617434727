"""oracle/torso_grid.py -- TEST INFRASTRUCTURE (CPU checker of the torso occupancy-grid refresh; never imported by the product path).

CPU fp32 restatement of RADNeRFTorso.update_extra_state (modules/radnerfs/radnerf_torso.py:201-242) and
RADNeRFTorsowithSR.update_extra_state (radnerf_torso_sr.py:246-288) on top of oracle.render.OracleModel.forward_torso /
forward_torso_sr.  Pinned against the reference's own methods by oracle/make_torso_grid_golden.py (tests/golden/torso_*grid*.npz).

Noise is an explicit [H,H,2] tensor in [0,1): the reference's `torch.rand_like` draws of radnerf_torso.py:227 in its
meshgrid(x, y) order (one chunk when S >= grid_size, which is how the goldens are made: the field is then evaluated in one batch
as in the reference).
"""
import torch
import torch.nn.functional as F


def raw_grid(orc, noise, pose6=None, code=None, lm68=None):
    """Step 1 of the refresh (radnerf_torso.py:204-233): alpha at every cell, [H*H] at the reference's transposed index y*H + x.
    The torso-SR field (lm68 given) sees image = weights_sum = 0, as the reference passes it."""
    H = orc.grid_size
    r = torch.arange(H, dtype=torch.int32)
    xx, yy = torch.meshgrid(r, r, indexing="ij")
    coords = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1)], dim=-1)
    idx = (coords[:, 1] * H + coords[:, 0]).long()
    hgs = 1 / H
    xys = 2 * coords.float() / (H - 1) - 1
    xys = xys * (1 - hgs)
    xys += (noise.reshape(-1, 2) * 2 - 1) * hgs
    c = None if code is None else code.reshape(1, -1)
    if lm68 is None:
        alphas, _, _ = orc.forward_torso(xys, pose6.reshape(1, 6), c)
    else:
        n = xys.shape[0]
        alphas, _, _ = orc.forward_torso_sr(xys, None, c, torch.zeros(n, 3), torch.zeros(n, 1), lm68.reshape(1, 136))
    tmp = torch.zeros(H * H)
    tmp[idx] = alphas.squeeze(1).float()
    return tmp


def update_extra_state(orc, noise, grid0, decay=0.95, pose6=None, code=None, lm68=None):
    """radnerf_torso.py:204-242.  Returns (raw grid, new density_grid_torso, mean_density_torso); grid0 is not modified."""
    H = orc.grid_size
    tmp = raw_grid(orc, noise, pose6, code, lm68)
    dil = F.max_pool2d(tmp.view(1, 1, H, H), kernel_size=5, stride=1, padding=2).view(-1)
    grid = torch.maximum(grid0.float() * decay, dil)
    return tmp, grid, torch.mean(grid).item()
