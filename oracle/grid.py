"""oracle/grid.py -- TEST INFRASTRUCTURE (CPU checker of the occupancy-grid maintenance; never imported by the product path).

CPU fp32 restatement of NeRFRenderer.update_extra_state (head grid) and mark_untrained_grid
(modules/radnerfs/renderer.py:131-284) on top of oracle.render.OracleModel and the C restatement of
morton3D / morton3D_dilation / packbits (oracle/native_ops.c).  Pinned against the reference's own
methods by oracle/make_grid_golden.py (tests/golden/grid_*.npz).

Noise is an explicit [C,H,H,H,3] tensor in [0,1): the reference's `torch.rand_like` draws of
renderer.py:258 in its meshgrid(x,y,z) order (one chunk per cascade when S >= grid_size).
"""
import torch

from . import ops
from .render import _mlp


def density(orc, xyzs, cond_feat):
    """RADNeRF.density (radnerf.py:143-166): -> (sigma [n], geo_feat [n,128])."""
    st = orc.st
    n = xyzs.shape[0]
    cond = cond_feat.reshape(1, -1).repeat([n, 1])
    pos = orc._grid(xyzs, orc.bound, "position_embedder.embeddings", "position_embedder.offsets", orc.per_level_scale)
    amb = _mlp(torch.cat([pos, cond], dim=1), [st[f"ambient_net.net.{i}.weight"] for i in range(orc.hp["num_layers_ambient"])], orc._linear)
    amb = orc._grid(torch.tanh(amb.float()), 1, "ambient_embedder.embeddings", "ambient_embedder.offsets", orc.per_level_scale_amb)
    h = _mlp(torch.cat([pos, amb], dim=-1), [st[f"sigma_net.net.{i}.weight"] for i in range(orc.hp["num_layers_sigma"])], orc._linear)
    return torch.exp(h[..., 0].float()), h[..., 1:]


def cell_coords(H):
    """[H^3, 3] int32 cell coordinates in meshgrid(x, y, z) order (renderer.py:243-244, one chunk)."""
    r = torch.arange(H, dtype=torch.int32)
    xx, yy, zz = torch.meshgrid(r, r, r, indexing="ij")
    return torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], dim=-1)


def cascade_bound(orc, cas):
    bound = min(2 ** cas, orc.bound)
    return bound, bound / orc.grid_size


def raw_grid(orc, cond_feat, noise):
    """Steps 1 of the refresh (renderer.py:231-264): sigma * density_scale at every cell, [C, H^3] in Morton order."""
    H, C = orc.grid_size, orc.cascade
    coords = cell_coords(H)
    idx = ops.morton3D(coords).long()
    xyzs = 2 * coords.float() / (H - 1) - 1
    tmp = torch.zeros(C, H ** 3)
    for cas in range(C):
        bound, hgs = cascade_bound(orc, cas)
        cas_xyzs = xyzs * (bound - hgs)
        cas_xyzs += (noise[cas].reshape(-1, 3) * 2 - 1) * hgs
        sig, _ = density(orc, cas_xyzs, cond_feat)
        sig = sig.reshape(-1) * orc.density_scale
        tmp[cas, idx] = sig
    return tmp


def update_extra_state(orc, cond_feat, noise, density_grid, decay=0.95, density_thresh=10.0):
    """renderer.py:230-278.  Returns (raw grid, new density_grid, mean_density, bitfield); density_grid is not modified."""
    tmp = raw_grid(orc, cond_feat, noise)
    dil = ops.morton3D_dilation(tmp)
    grid = density_grid.clone().float()
    valid = (grid >= 0) & (dil >= 0)
    grid[valid] = torch.maximum(grid[valid] * decay, dil[valid])
    mean = torch.mean(grid.clamp(min=0)).item()
    bits = ops.packbits(grid, min(mean, density_thresh))
    return tmp, grid, mean, bits


def mark_untrained_grid(orc, density_grid, poses, intrinsic, S=64):
    """renderer.py:131-199 on the CPU (one chunk of cells, S poses at a time).  Returns the marked copy of density_grid."""
    H, C = orc.grid_size, orc.cascade
    fx, fy, cx, cy = intrinsic
    coords = cell_coords(H)
    idx = ops.morton3D(coords).long()
    world = (2 * coords.float() / (H - 1) - 1).unsqueeze(0)
    B = poses.shape[0]
    count = torch.zeros(C, H ** 3)
    for cas in range(C):
        bound, hgs = cascade_bound(orc, cas)
        cw = world * (bound - hgs)
        for head in range(0, B, S):
            tail = min(head + S, B)
            cam = cw - poses[head:tail, :3, 3].unsqueeze(1)
            cam = cam @ poses[head:tail, :3, :3]
            mz = cam[:, :, 2] > 0
            mx = torch.abs(cam[:, :, 0]) < cx / fx * cam[:, :, 2] + hgs * 2
            my = torch.abs(cam[:, :, 1]) < cy / fy * cam[:, :, 2] + hgs * 2
            count[cas, idx] += (mz & mx & my).sum(0).reshape(-1).float()
    out = density_grid.clone().float()
    out[count == 0] = -1
    return out
