"""tools/grid_half_bench.py -- the grid encoder on half tables (gfpp.h section (L)) timed beside the reference's compiled half kernels
and libgfpp's fp32 grid ops, in one process, on the same inputs.  Prints one JSON line.

    python tools/grid_half_bench.py [--points 390784] [--reps 20]

The shapes of one head training step's grid calls (390 784 sample points): the position grid (D = 3) of the May configuration and a
2-D ambient grid (radnerf/base.yaml's ambient_coord_dim), 16 levels x 2 channels, tiled, linear.  Legs per grid (CUDA events, median of `reps` after two warm-up
calls; ms per call):
  * forward with dy_dx (grid_encode_forward with calc_grad_inputs);
  * backward: table gradient (f16x2 / float2 reductions into a zeroed table) and input gradient through dy_dx.
Each leg runs on libgfpp's half ops (through the level-B shims, as the reference's Python calls them), on the reference's own
half kernels (oracle/_ref/_gridencoder, when it was built) and on libgfpp's fp32 ops (fp32 table, outputs and gradients).  The
table zeroing that grid.py does before the backward (torch.zeros_like) is outside the timed window.
Bytes per leg are counted from shapes (inputs, outputs, dy_dx, upstream gradient) plus 2^D corner gathers / reductions of one
table entry per (point, level); the achieved rate is reported against the H100 SXM's 3.35 TB/s only as a ratio of that count.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _median_ms(fn, reps):
    fn()
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def _ref_module():
    so = os.path.join(ROOT, "oracle", "_ref", "_gridencoder", "_gridencoder.so")
    if not os.path.exists(so):
        return None
    spec = importlib.util.spec_from_file_location("_gridencoder", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # the card's name still comes from torch
        return f"{torch.cuda.get_device_name()} (nvidia-smi: {e})"


def bench_grid(name, lay, B, mods, reps):
    dev = "cuda"
    D, L = lay.input_dim, lay.num_levels
    g = torch.Generator().manual_seed(1)
    x = torch.rand(B, D, generator=g).to(dev)
    emb32 = (torch.randn(lay.n_entries, 2, generator=g) * 0.1).to(dev)
    off = torch.from_numpy(lay.offsets).to(dev)
    S, H = float(lay.S), lay.base_resolution
    grad32 = (torch.randn(L, B, 2, generator=g) * 0.05).to(dev)
    res = {"points": B, "D": D, "levels": L, "table_entries": lay.n_entries}
    outs = {}
    for label, ge, dt in mods:
        emb = emb32.to(dt)
        grad = grad32.to(dt)
        out = torch.empty(L, B, 2, dtype=dt, device=dev)
        dd = torch.empty(B, L * D * 2, dtype=dt, device=dev)
        gemb = torch.zeros_like(emb)
        gi = torch.zeros(B, D, dtype=dt, device=dev)
        fwd = lambda: ge.grid_encode_forward(x, emb, off, out, B, D, 2, L, S, H, dd, lay.gridtype_id, False, lay.interp_id)   # noqa: E731
        bwd = lambda: ge.grid_encode_backward(grad, x, emb, off, gemb, B, D, 2, L, S, H, dd, gi, lay.gridtype_id, False,      # noqa: E731
                                              lay.interp_id)
        t_f = _median_ms(fwd, reps)
        ts = []
        for _ in range(reps):
            gemb.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            bwd()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        t_b = float(np.median(ts))
        es = torch.finfo(dt).bits // 8
        b_f = B * D * 4 + L * B * 2 * es * (1 + D) + B * L * (1 << D) * 2 * es      # inputs, outputs + dy_dx, corner gathers
        b_b = B * D * 4 + L * B * 2 * es + B * L * (1 << D) * 2 * es * 2 + (L * B * 2 * es + B * L * D * 2 * es + B * D * es)
        res[label] = {"forward_dydx_ms": round(t_f, 4), "backward_table_and_input_ms": round(t_b, 4),
                      "forward_bytes_per_s_over_3.35TB/s": round(b_f / (t_f * 1e-3) / 3.35e12, 4),
                      "backward_bytes_per_s_over_3.35TB/s": round(b_b / (t_b * 1e-3) / 3.35e12, 4)}
        outs[label] = (out.clone(), dd.clone(), gi.clone())
    if "ours_half" in outs and "reference_half" in outs:
        res["ours_half_bit_equal_reference_half"] = all(torch.equal(a.view(torch.int16), b.view(torch.int16))
                                                        for a, b in zip(outs["ours_half"], outs["reference_half"]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=390_784)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "grid_half_bench needs a GPU"
    from genefaceplusplus_b200 import backend_shims
    from genefaceplusplus_b200.config import GridLayout, may_hparams
    hp = may_hparams()          # the 2-D ambient grid of radnerf/base.yaml (ambient_coord_dim 2); lm3d_radnerf.yaml's is 3-D
    gt = {"tiledgrid": "tiled", "hashgrid": "hash"}[hp["grid_type"]]
    it = hp["grid_interpolation_type"]
    pos = GridLayout(3, log2_hashmap_size=hp["log2_hashmap_size"], desired_resolution=hp["desired_resolution"] * hp["bound"], gridtype=gt,
                     interpolation=it)
    amb = GridLayout(2, log2_hashmap_size=hp["log2_hashmap_size"], desired_resolution=hp["desired_resolution"],
                     gridtype=gt, interpolation=it)
    ours = backend_shims.make_modules()["_gridencoder"]
    ref = _ref_module()
    mods = [("ours_half", ours, torch.float16)] + ([("reference_half", ref, torch.float16)] if ref is not None else []) + \
           [("ours_fp32", ours, torch.float32)]
    line = {"what": "grid encoder at one head training step's size: libgfpp half ops (gfpp.h section L) vs the reference's half kernels "
                    "vs libgfpp fp32 ops, same inputs, same process",
            "gpu": _gpu_info(), "reference_built": ref is not None,
            "position_grid": bench_grid("position", pos, a.points, mods, a.reps),
            "ambient_grid": bench_grid("ambient", amb, a.points, mods, a.reps)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
