"""Shared helpers of the GPU parity tests."""
import math

import numpy as np
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import GridLayout
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso


def lively_state(state, gain=4.0):
    """Scale the three head MLPs so the field has O(1) dynamic range (sigma 0.1..5, colours 0..1, ambient
    coordinates spanning [-1,1]).  The default-init scene of SURVEY.md 8(d) is very bland (colours 0.49..0.51),
    which would let real bugs hide below 1e-3; the lively variant makes them glaring."""
    out = dict(state)
    for k in list(out):
        if k.startswith(("ambient_net", "sigma_net", "color_net", "torso_deform_net", "torso_canonicial_net")):
            out[k] = out[k] * gain
    return out


def build_model(sc: scn.Scene, state=None, device="cuda", precision="fp32"):
    cls = RADNeRFTorso if sc.torso else RADNeRF
    m = cls(sc.hparams)
    m.mlp_precision = precision
    m.load_state_dict(state if state is not None else sc.state, strict=True)
    m.density_scale = sc.density_scale
    return m.to(device).eval()


def relu_ties(trace, flip_band):
    """Points within flip_band (relative to the layer's largest pre-activation) of a ReLU tie in any of the five ReLU layers of an
    oracle forward's trace: a last-bit difference between two implementations can flip such a ReLU."""
    tie = torch.zeros(trace["relu_pre"][0].shape[0], dtype=torch.bool)
    for pre in trace["relu_pre"]:
        tie |= (pre.abs() < flip_band * pre.abs().max()).any(1)
    return tie


def _ambient_levels(amb, hp):
    """(scale, pos = u * scale + 0.5) per level of the ambient grid for ambient coordinates amb [N,A] in [-1,1], u = (amb + 1) / 2,
    in float64."""
    lay = GridLayout(amb.shape[1], log2_hashmap_size=hp["log2_hashmap_size"], desired_resolution=hp["desired_resolution"])
    u = (amb.detach().double() + 1) / 2
    for lv in range(lay.num_levels):
        scale = float(np.exp2(np.float32(lv) * lay.S) * np.float32(lay.base_resolution) - np.float32(1.0))
        yield scale, u * scale + 0.5


def ties(trace, amb, hp, flip_band, cell_band):
    """(points at a ReLU tie (relu_ties), points whose ambient coordinate lies within cell_band of a cell face of any level of the
    ambient grid), from an oracle forward's trace and ambient output."""
    face = torch.zeros(amb.shape[0], dtype=torch.bool)
    for scale, pos in _ambient_levels(amb, hp):
        face |= ((pos - pos.round()).abs() < cell_band * scale).any(1)
    return relu_ties(trace, flip_band), face


def cell_flips(amb_a, amb_b, hp):
    """Points whose two ambient coordinates [N,A] fall into different cells of some level of the ambient grid, where the grid's
    input gradient (a per-cell slope) jumps.  The cell is floor(u * scale + 0.5) with u = (amb + 1) / 2, in the fp32 arithmetic of
    the grid kernels and of the C checker."""
    lay = GridLayout(amb_a.shape[1], log2_hashmap_size=hp["log2_hashmap_size"], desired_resolution=hp["desired_resolution"])
    ua, ub = (amb_a.detach().float() + 1) / 2, (amb_b.detach().float() + 1) / 2
    flip = torch.zeros(amb_a.shape[0], dtype=torch.bool)
    for lv in range(lay.num_levels):
        scale = torch.tensor(np.exp2(np.float32(lv) * np.float32(lay.S)) * np.float32(lay.base_resolution) - np.float32(1.0), dtype=torch.float32)
        flip |= (torch.floor(ua * scale + 0.5) != torch.floor(ub * scale + 0.5)).any(1)
    return flip


def psnr(a, b):
    mse = ((a.double() - b.double()) ** 2).mean().item()
    return float("inf") if mse == 0 else 10 * math.log10(1.0 / mse)


def parity_report(mine, ref, knife=None, knife_tol=1e-3, tol=1e-3):
    """max-abs / PSNR of `mine` vs the oracle `ref` ([N,3] or [N]).

    Rays whose transmittance came within `knife_tol` (relative) of T_thresh in the oracle are "knife-edge":
    an fp32 reordering can legitimately flip their termination, which adds or drops one sample of weight
    <= T_thresh.  They are REPORTED (count) and excluded from the max-abs bar, never silently masked;
    the PSNR is computed over ALL pixels."""
    d = (mine.float().cpu() - ref.float().cpu()).abs()
    if d.dim() > 1:
        d = d.reshape(d.shape[0], -1).max(-1).values
    d = torch.nan_to_num(d, nan=0.0)  # NaN == NaN positions (depth of rays that miss the aabb) are checked separately
    excl = torch.zeros_like(d, dtype=torch.bool) if knife is None else (knife.cpu().reshape(-1) < knife_tol)
    worst = d[~excl].max().item() if (~excl).any() else 0.0
    return {"max_abs": worst, "max_abs_all": d.max().item(), "n_knife": int(excl.sum()), "n_over": int((d > tol).sum()),
            "psnr": psnr(torch.nan_to_num(mine.float().cpu()), torch.nan_to_num(ref.float().cpu()))}
