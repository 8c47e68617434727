"""tools/train_bench.py -- the training-side native ops of libgfpp (csrc/train_kernels.cu; SURVEY 8(f) rank 4) timed beside the
REFERENCE'S OWN training kernels (oracle/_ref, compiled unmodified) on the same inputs, same box, same run: one training step's
worth of marching, compositing forward + backward and grid-encoder backward on the rays of one 256x256 frame of the bench scene
(N = 65 536 rays, max_steps 16; what `RADNeRFTask.run_model` marches per step is 4 096-65 536 rays).

    python tools/train_bench.py [--size 256] [--reps 5]

`measure()` is also what bench.py calls for the `train_ops` object of its JSON line.  Every call below uses exactly the argument
lists tests/test_gpu_train_ops.py validated on the GPU (ours through the backend shims, the reference's through its pybind
modules)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def measure(size=256, reps=5):
    from genefaceplusplus_b200 import backend_shims, scene as scn
    from genefaceplusplus_b200.config import GridLayout
    from oracle import gpu_ref_ops
    ours = backend_shims.make_modules()
    have_ref = all(os.path.exists(os.path.join(ROOT, "oracle", "_ref", n, n + ".so")) for n in ("_raymarching_face", "_gridencoder"))
    ref_rm = gpu_ref_ops._load("_raymarching_face") if have_ref else None
    ref_ge = gpu_ref_ops._load("_gridencoder") if have_ref else None
    sc = scn.Scene(H=size, W=size, T=2, torso=False)
    fi = sc.frame_inputs(1)
    ro, rd = fi["rays_o"].view(-1, 3).contiguous().cuda(), fi["rays_d"].view(-1, 3).contiguous().cuda()
    N, max_steps = ro.shape[0], 16
    aabb, bits = sc.state["aabb_infer"].cuda(), sc.state["density_bitfield"].cuda()
    nears, fars = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
    ours["_raymarching_face"].near_far_from_aabb(ro, rd, aabb, N, 0.05, nears, fars)
    M = N * max_steps
    noises = torch.zeros(N, device="cuda")
    res = {"workload": f"{N} rays (one {size}x{size} frame of the bench scene), max_steps {max_steps}", "reps": reps,
           "note": "CUDA events, median; ms per call; `ref` = the reference's own kernels (oracle/_ref) on the same inputs"}

    def march(mod):
        xyzs, dirs, deltas = torch.zeros(M, 3, device="cuda"), torch.zeros(M, 3, device="cuda"), torch.zeros(M, 2, device="cuda")
        rays = torch.empty(N, 3, dtype=torch.int32, device="cuda")
        counter = torch.zeros(2, dtype=torch.int32, device="cuda")

        def run():
            counter.zero_()
            mod.march_rays_train(ro, rd, bits, 1.0, 1 / 256, max_steps, N, 1, 128, M, nears, fars, xyzs, dirs, deltas, rays, counter, noises)
        return run, (xyzs, dirs, deltas, rays, counter)

    run_o, (xyzs, dirs, deltas, rays, counter) = march(ours["_raymarching_face"])
    res["march_rays_train_ms"] = _median_ms(run_o, reps)
    m = int(counter[0].item())
    res["points"] = m
    if have_ref:
        run_r, _ = march(ref_rm)
        res["march_rays_train_ref_ms"] = _median_ms(run_r, reps)
    # compositing on OUR (deterministic) layout for both implementations
    g = torch.Generator(device="cuda").manual_seed(0)
    sig = torch.rand(M, device="cuda", generator=g) * 6
    rgb = torch.rand(M, 3, device="cuda", generator=g)
    amb = torch.rand(M, device="cuda", generator=g)
    ws, asum, depth, image = torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, device="cuda"), torch.empty(N, 3, device="cuda")
    gws, gas, gim = torch.randn(N, device="cuda", generator=g), torch.randn(N, device="cuda", generator=g), torch.randn(N, 3, device="cuda", generator=g)
    gs, gr, ga = torch.zeros(M, device="cuda"), torch.zeros(M, 3, device="cuda"), torch.zeros(M, device="cuda")
    for tag, mod in (("", ours["_raymarching_face"]), ("_ref", ref_rm)):
        if mod is None:
            continue
        res[f"composite_rays_train_forward{tag}_ms"] = _median_ms(
            lambda: mod.composite_rays_train_forward(sig, rgb, amb, deltas, rays, M, N, 1e-4, ws, asum, depth, image), reps)
        res[f"composite_rays_train_backward{tag}_ms"] = _median_ms(
            lambda: mod.composite_rays_train_backward(gws, gas, gim, sig, rgb, amb, deltas, rays, ws, asum, image, M, N, 1e-4, gs, gr, ga), reps)
    # grid encoder: forward with dy_dx + backward on the marched points (position grid of the May config)
    lay = GridLayout(3, log2_hashmap_size=16, desired_resolution=2048, gridtype="tiled")
    offsets = torch.from_numpy(np.asarray(lay.offsets, dtype=np.int32)).cuda()
    table = sc.state["position_embedder.embeddings"].cuda().contiguous()
    B = max(128, m)
    x01 = ((xyzs[:B] + 1) / 2).contiguous()
    S = float(np.log2(lay.per_level_scale))
    grad = torch.randn(16, B, 2, device="cuda", generator=g)
    out, dy = torch.empty(16, B, 2, device="cuda"), torch.empty(B, 16 * 3 * 2, device="cuda")
    ge_, gi_ = torch.zeros_like(table), torch.zeros(B, 3, device="cuda")
    for tag, mod in (("", ours["_gridencoder"]), ("_ref", ref_ge)):
        if mod is None:
            continue
        res[f"grid_encode_forward_dydx{tag}_ms"] = _median_ms(lambda: mod.grid_encode_forward(x01, table, offsets, out, B, 3, 2, 16, S, 16, dy, 1, False, 0), reps)
        res[f"grid_encode_backward{tag}_ms"] = _median_ms(
            lambda: mod.grid_encode_backward(grad, x01, table, offsets, ge_, B, 3, 2, 16, S, 16, dy, gi_, 1, False, 0), reps)
    res["grid_points"] = B
    if not have_ref:
        res["ref"] = "oracle/_ref/*.so not present"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(measure(a.size, a.reps)))


if __name__ == "__main__":
    main()
