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
only) and 2 grids x 16 levels x 8 corners x 8 B = 2048 B of gathers per point.
Torso legs (the torso models' update_extra_state, radnerf_torso.py:201-242 / radnerf_torso_sr.py:246-288), 128^2 = 16 384 cells:
  * native refresh of density_grid_torso for RADNeRFTorso and RADNeRFTorsowithSR (frame-bias fold -> k_torso_query /
    k_torso_sr_query -> k_torso_dilate_ema -> k_mean_thresh), including the one .item() of mean_density_torso; launches per call;
  * eager: the reference's procedure on the GPU -- forward_torso as PyTorch F.linear / ReLU over libgfpp's per-op freq / grid
    encoder kernels, then max_pool2d, maximum, mean().item().
  Algorithmic FLOP per cell: 2 x the multiply-adds of the deform and canonical nets (and the head-aware encoder), from the weights."""
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


def _mlp(x, net):
    for i, lin in enumerate(net.net):
        x = F.linear(x, lin.weight)
        if i != len(net.net) - 1:
            x = F.relu(x)
    return x


def eager_torso_refresh(m, enc, cond, code, noise, decay):
    """radnerf_torso.py:204-242 (radnerf_torso_sr.py:249-288 when m is a torso-SR model) with S >= grid_size: one chunk of cells,
    forward_torso as PyTorch ops over libgfpp's per-op encoder kernels."""
    H = m.grid_size
    r = torch.arange(H, dtype=torch.int32, device="cuda")
    xx, yy = torch.meshgrid(r, r, indexing="ij")
    coords = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1)], dim=-1)
    idx = (coords[:, 1] * H + coords[:, 0]).long()
    xys = (2 * coords.float() / (H - 1) - 1) * (1 - 1 / H) + (noise.view(-1, 2) * 2 - 1) * (1 / H)
    if cond.numel() == 136:     # torso-SR model: its host-side forward_torso over the same per-op encoders (m.encoders)
        alphas, _, _ = m.forward_torso(xys, None, code.view(1, -1), lm68=cond)
    else:
        x = xys * m.torso_shrink
        n = x.shape[0]
        h = torch.cat([enc.freq_encode(x, 10), enc.freq_encode(cond.view(1, 6), 4).expand(n, -1), code.view(1, -1).expand(n, -1)], -1)
        dx = _mlp(h, m.torso_deform_net)
        lay = m.torso_embedder.layout
        xf = enc.grid_encode(((x + dx).clamp(-1, 1) + 1) / 2, m.torso_embedder.embeddings, m.torso_embedder.offsets, lay.per_level_scale,
                             lay.base_resolution, 1, False, 0)
        alphas = torch.sigmoid(_mlp(torch.cat([xf, h], -1), m.torso_canonicial_net)[..., :1])
    tmp = torch.zeros(H * H, device="cuda")
    tmp[idx] = alphas.squeeze(1).float()
    tmp = F.max_pool2d(tmp.view(1, 1, H, H), kernel_size=5, stride=1, padding=2).view(-1)
    m.density_grid_torso = torch.maximum(m.density_grid_torso * decay, tmp)
    return torch.mean(m.density_grid_torso).item()


def measure_torso(res, reps):
    from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR, _NativeEncoders
    from genefaceplusplus_b200.scene import convert_poses
    from oracle import make_torso_grid_golden as mtg
    enc = _NativeEncoders()
    for kind in ("torso", "torso_sr"):
        inp = mtg.inputs(kind, 128)
        m = (RADNeRFTorsowithSR if kind == "torso_sr" else RADNeRFTorso)(inp["hp"])
        m.load_state_dict(inp["state"], strict=True)
        m = m.cuda().eval()
        m.encoders = enc
        nets = [m.torso_deform_net, m.torso_canonicial_net] + ([m.head_color_weights_encoder] if kind == "torso_sr" else [])
        macs = sum(p.numel() for net in nets for n_, p in net.named_parameters() if n_.endswith("weight"))
        cond = (inp["lm68s"][mtg.POSE_INDEX] if kind == "torso_sr" else convert_poses(inp["poses"][mtg.POSE_INDEX].view(1, 4, 4)).view(6)).cuda()
        code, noise = inp["code"].cuda(), inp["noise"].cuda()
        g0 = m.density_grid_torso.clone()
        ms = _median_ms(lambda: m.refresh_torso_grid(cond, code, noise, 0.95).item(), reps)
        res[f"{kind}_cells"] = 128 * 128
        res[f"{kind}_algorithmic_mflop"] = round(128 * 128 * 2 * macs / 1e6, 1)
        res[f"{kind}_native_refresh_ms"] = round(ms, 3)
        res[f"{kind}_native_launches_per_call"] = m.last_launch_count
        m.density_grid_torso.copy_(g0)
        with torch.no_grad():
            res[f"{kind}_eager_libgfpp_ops_ms"] = round(_median_ms(lambda: eager_torso_refresh(m, enc, cond, code, noise, 0.95), reps), 3)


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
    measure_torso(res, reps)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(measure(a.reps)))


if __name__ == "__main__":
    main()
