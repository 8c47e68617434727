"""tools/grid_bench.py -- the occupancy-grid refresh (update_extra_state's device half) and the density query of libgfpp timed beside
an eager restatement of the reference's procedure, same inputs, same run.  Prints one JSON line.

    python tools/grid_bench.py [--reps 5]

Legs (CUDA events, median of `reps` after one warm-up call; ms per call):
  * native refresh of the 128^3 head grid (k_density -> k_dilate_ema -> k_mean_thresh -> k_packbits_dev -> packed occupancy),
    including the one device-to-host read of mean_density, as update_extra_state does it; models packed in the fp16 and fp32 modes
    (the density query runs the same fp32 field in both);
  * density() at 2^21 points (sigma + geo_feat);
  * eager: renderer.py:243-278 as the reference runs it on the GPU -- PyTorch F.linear / ReLU / tanh / exp under fp16 autocast over
    per-op grid_encode_forward launches, then the per-op morton3D_dilation, the masked EMA, mean().item() and packbits -- once over
    libgfpp's per-op kernels and, where oracle/_ref was built, once over the reference's own compiled kernels.
Algorithmic work of one refresh: C*H^3 points x (96*128 + 128*128 + 128*3 + 64*128 + 128*128 + 128*1) * 2 FLOP (the sigma column
only) and 2 grids x 16 levels x 8 corners x 8 B = 2048 B of gathers per point."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FLOP_PER_POINT = 2 * (96 * 128 + 128 * 128 + 128 * 3 + 64 * 128 + 128 * 128 + 128 * 1)
GATHER_BYTES_PER_POINT = 2 * 16 * 8 * 8


def _median_ms(fn, reps):
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
    return sorted(ts)[len(ts) // 2]


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the numbers are still measured; say that the card could not be read
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})"}


def eager_refresh(model, ge, rm, cond_feat, noise, decay, autocast=True):
    """renderer.py:231-278 with S >= grid_size (one chunk), C = 1, the field as PyTorch ops over per-op grid-encoder kernels."""
    dev = "cuda"
    H = model.grid_size
    st = {k: v for k, v in model.state_dict().items()}
    r = torch.arange(H, dtype=torch.int32, device=dev)
    xx, yy, zz = torch.meshgrid(r, r, r, indexing="ij")
    coords = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1).contiguous()
    N = coords.shape[0]
    idx = torch.empty(N, dtype=torch.int32, device=dev)
    rm.morton3D(coords, N, idx)
    xyzs = 2 * coords.float() / (H - 1) - 1
    bound, hgs = 1.0, 1.0 / H
    x = xyzs * (bound - hgs) + (noise.view(-1, 3) * 2 - 1) * hgs
    pos_l, amb_l = model.position_embedder.layout, model.ambient_embedder.layout

    def genc(x01, emb, off, lay):
        out = torch.empty(16, N, 2, device=dev)
        ge.grid_encode_forward(x01.contiguous(), emb, off, out, N, lay.input_dim, 2, 16, float(np.log2(lay.per_level_scale)),
                               lay.base_resolution, None, lay.gridtype_id, False, lay.interp_id)
        return out.permute(1, 0, 2).reshape(N, 32)

    with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
        pos = genc((x + 1) / 2, st["position_embedder.embeddings"], st["position_embedder.offsets"], pos_l)
        h = torch.cat([pos, cond_feat.view(1, -1).expand(N, -1)], 1)
        h = F.relu(F.linear(h, st["ambient_net.net.0.weight"]))
        h = F.relu(F.linear(h, st["ambient_net.net.1.weight"]))
        amb = torch.tanh(F.linear(h, st["ambient_net.net.2.weight"]).float())
        af = genc((amb + 1) / 2, st["ambient_embedder.embeddings"], st["ambient_embedder.offsets"], amb_l)
        h = F.relu(F.linear(torch.cat([pos, af], -1), st["sigma_net.net.0.weight"]))
        h = F.relu(F.linear(h, st["sigma_net.net.1.weight"]))
        h = F.linear(h, st["sigma_net.net.2.weight"])
        sigma = torch.exp(h[..., 0].float())
    tmp = torch.zeros(1, N, device=dev)
    tmp[0, idx.long()] = sigma * model.density_scale
    dil = torch.empty_like(tmp)
    rm.morton3D_dilation(tmp, 1, H, dil)
    grid = model.density_grid
    valid = (grid >= 0) & (dil >= 0)
    grid[valid] = torch.maximum(grid[valid] * decay, dil[valid])
    mean = torch.mean(grid.clamp(min=0)).item()
    rm.packbits(grid, N // 8, min(mean, model.density_thresh), model.density_bitfield)
    return mean


def measure(reps=5):
    from genefaceplusplus_b200 import backend_shims
    from oracle import make_grid_golden as mg
    res = {"workload": "head grid 128^3 (cascade 1) of the synthetic May-architecture model, density_scale 8, decay 0.95",
           "reps": reps, "note": "CUDA events, median, ms per call; refresh legs include the mean_density device-to-host read"}
    res.update(_gpu_info())
    H = 128
    pts = H ** 3
    res["points"] = pts
    res["algorithmic_gflop"] = round(pts * FLOP_PER_POINT / 1e9, 1)
    res["algorithmic_gather_gb"] = round(pts * GATHER_BYTES_PER_POINT / 1e9, 2)
    g = np.load(os.path.join(ROOT, "tests", "golden", "grid_head128.npz"))
    cf = torch.from_numpy(g["cond_feat"]).cuda()
    for prec in ("fp16", "fp32"):
        from genefaceplusplus_b200.renderer import RADNeRF
        inp = mg.inputs(H)
        m = RADNeRF(inp["hp"])
        m.load_state_dict(inp["state"], strict=True)
        m.density_scale, m.mlp_precision = mg.DS, prec
        m = m.cuda().eval()
        noise = inp["noise"].cuda()
        ms = _median_ms(lambda: m.refresh_density_grid(cf, noise, mg.DECAY).item(), reps)
        res[f"native_refresh_{prec}_ms"] = round(ms, 3)
        res[f"native_refresh_{prec}_tflops"] = round(pts * FLOP_PER_POINT / ms / 1e9, 2)
    x = (torch.rand(1 << 21, 3, device="cuda") * 2 - 1)
    res["density_2e21_ms"] = round(_median_ms(lambda: m.density(x, cf), reps), 3)
    mods = backend_shims.make_modules()
    res["eager_libgfpp_ops_ms"] = round(_median_ms(lambda: eager_refresh(m, mods["_gridencoder"], mods["_raymarching_face"], cf, noise, mg.DECAY), reps), 3)
    have_ref = all(os.path.exists(os.path.join(ROOT, "oracle", "_ref", n, n + ".so")) for n in ("_raymarching_face", "_gridencoder"))
    if have_ref:
        from oracle import gpu_ref_ops
        ref_rm, ref_ge = gpu_ref_ops._load("_raymarching_face"), gpu_ref_ops._load("_gridencoder")
        res["eager_reference_kernels_ms"] = round(_median_ms(lambda: eager_refresh(m, ref_ge, ref_rm, cf, noise, mg.DECAY), reps), 3)
    else:
        res["eager_reference_kernels_ms"] = "oracle/_ref/*.so not present"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(measure(a.reps)))


if __name__ == "__main__":
    main()
