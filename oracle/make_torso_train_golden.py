"""oracle/make_torso_train_golden.py -- pins the training torso field and the torso training step against the reference's OWN
RADNeRFTorso (modules/radnerfs/radnerf_torso.py) and its backward, and writes tests/golden/train_torso.npz.

Runs only where the reference sources exist.  The reference's RADNeRFTorso is built from egs/datasets/May/lm3d_radnerf_torso.yaml,
loads the synthetic May torso scene of oracle/torso_train.golden_scene() (32x32, deform output layer scaled by DEFORM_GAIN) with
strict=True and runs on the CPU in .train() mode through oracle/ref_shim.py plus oracle/ref_train_shim.py.
  (a) forward_torso at GOLDEN_M seeded points (some where shrink * x + dx leaves [-1, 1]) for pose frame GOLDEN_FRAME and code row
      torso_individual_codes[index] (index a [1] tensor, as the task passes it), then backward of a seeded linear loss of alpha, color
      and dx;
  (b) render() in training mode, perturb=False, max_steps 16, then backward of the task's loss for torso_train_mode 1 (MSE of
      torso_rgb_map against a seeded target plus lambda_weights_entropy times the alpha entropy).
The same computations through oracle/torso_train.py (the checker) are compared with it and the differences printed.

Stored for both parts: the inputs, the outputs, the reference's fp32 gradients of the six torso weights and of the code row, the table
gradient at N_SAMPLE seeded entries and its per-level L2 norms, and the same gradients from the checker with float64 dense layers.

Usage:  python -m oracle.make_torso_train_golden
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import field_train as ft  # noqa: E402
from oracle import ops, ref_shim, ref_train_shim  # noqa: E402
from oracle import torso_train as tt  # noqa: E402

N_SAMPLE = 2048
WEIGHTS = tt.TRAINABLE[:6]


def table_sample(n_entries):
    return np.sort(np.random.Generator(np.random.PCG64(23)).choice(n_entries, N_SAMPLE, replace=False)).astype(np.int64)


def level_norms(grad, offsets):
    off = offsets.tolist()
    return np.asarray([float(grad[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)], dtype=np.float64)


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def linear_loss(a, c, dx, coef):
    return (a * coef[1].to(a.dtype)).sum() + (c * coef[2].to(c.dtype)).sum() + (dx * coef[3].to(dx.dtype)).sum()


def store_grads(g, prefix, grads, code_grad, table_grad, offsets, idx):
    for k in WEIGHTS:
        g[f"{prefix}.{k}"] = grads[k].detach().numpy().astype(np.float32)
    g[f"{prefix}.code"] = code_grad.detach().numpy().astype(np.float32)
    if table_grad is not None:
        g[f"{prefix}.table_sample"] = table_grad[idx].detach().numpy().astype(np.float32)
        g[f"{prefix}.table_level_norms"] = level_norms(table_grad, offsets)


def main():
    cwd = os.getcwd()
    ops.build()
    set_hparams = ref_shim.install(ops)
    ref_train_shim.install_training(ops)
    from modules.radnerfs.radnerf_torso import RADNeRFTorso
    sc = tt.golden_scene()
    hp = sc.hparams
    ref_hp = set_hparams("egs/datasets/May/lm3d_radnerf_torso.yaml", hparams_str="", print_hparams=False)
    for k in ("grid_size", "bound", "torso_shrink", "torso_individual_embedding_dim", "density_thresh_torso", "individual_embedding_dim"):
        assert ref_hp[k] == hp[k], (k, ref_hp[k], hp[k])
    assert int(ref_hp["torso_train_mode"]) == 1 and float(ref_hp["lambda_weights_entropy"]) == tt.LAMBDA_WEIGHTS_ENTROPY
    model = RADNeRFTorso(ref_hp)
    model.load_state_dict(sc.state, strict=True)
    model.density_scale = tt.GOLDEN_DS
    model.train()
    fi = sc.frame_inputs(tt.GOLDEN_FRAME)
    pose6 = fi["poses"]
    index = torch.tensor([tt.GOLDEN_INDEX])
    offsets = sc.state["torso_embedder.offsets"]
    n_entries = int(offsets[-1])
    idx = table_sample(n_entries)
    params = dict(model.named_parameters())
    report, g = {}, {}

    # ---- (a) forward_torso + backward at seeded points
    x, ca, cc, cd = tt.golden_points()
    coef = (x, ca, cc, cd)
    model.zero_grad(set_to_none=True)
    a, c, dx = model.forward_torso(x, pose6, model.torso_individual_codes[index])
    linear_loss(a, c, dx, coef).backward()
    p = tt.torso_params(sc.state)
    codes = sc.state["torso_individual_codes"].clone().requires_grad_(True)
    trace = {}
    oa, oc, odx = tt.torso_forward(p, hp, x, pose6, codes[index], trace)
    linear_loss(oa, oc, odx, coef).backward()
    n_out = int((trace["x_pre_clamp"].abs() > 1).any(-1).sum())
    for k, (r, o) in {"alpha": (a, oa), "color": (c, oc), "deform": (dx, odx)}.items():
        report[f"a.{k}"] = rel(o.detach(), r.detach())
    for k in tt.TRAINABLE:
        report[f"a.grad.{k}"] = rel(p[k].grad, params[k].grad)
    report["a.grad.code"] = rel(codes.grad[tt.GOLDEN_INDEX], params["torso_individual_codes"].grad[tt.GOLDEN_INDEX])
    g.update({"a.x": x.numpy(), "a.coef_alpha": ca.numpy(), "a.coef_color": cc.numpy(), "a.coef_deform": cd.numpy(), "pose6": pose6.numpy(),
              "a.alpha": a.detach().numpy(), "a.color": c.detach().numpy(), "a.deform": dx.detach().numpy()})
    store_grads(g, "a.grad", {k: params[k].grad for k in WEIGHTS}, params["torso_individual_codes"].grad[tt.GOLDEN_INDEX],
                params["torso_embedder.embeddings"].grad, offsets, idx)
    p64 = tt.torso_params(sc.state, torch.float64)
    codes64 = sc.state["torso_individual_codes"].double().clone().requires_grad_(True)
    linear_loss(*tt.torso_forward(p64, hp, x, pose6, codes64[index]), coef).backward()
    store_grads(g, "a.grad64", {k: p64[k].grad for k in WEIGHTS}, codes64.grad[tt.GOLDEN_INDEX], p64["torso_embedder.embeddings"].grad, offsets, idx)
    for k in WEIGHTS:
        report[f"a.fp32_vs_fp64.{k}"] = rel(params[k].grad, p64[k].grad)
    report["a.fp32_vs_fp64.code"] = rel(params["torso_individual_codes"].grad[tt.GOLDEN_INDEX], codes64.grad[tt.GOLDEN_INDEX])
    report["a.points_leaving"] = n_out

    # ---- (b) render() in training mode + the task's loss
    N = fi["rays_o"].numel() // 3
    gt = tt.golden_target(N)
    model.zero_grad(set_to_none=True)
    res = model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], pose6, index=index, dt_gamma=0, bg_color=fi["bg_color"],
                       perturb=False, force_all_rays=False, max_steps=tt.GOLDEN_MAX_STEPS)
    tt.task_loss(res, gt, tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    with torch.no_grad():
        cond_feat = model.cal_cond_feat(fi["cond"]).detach()
    hpar = ft.field_params(sc.state)
    p = tt.torso_params(sc.state)
    codes = sc.state["torso_individual_codes"].clone().requires_grad_(True)
    ind = sc.state["individual_embeddings"][index]
    orc = tt.train_step(hpar, p, hp, sc.state, fi["rays_o"], fi["rays_d"], cond_feat, ind, fi["bg_coords"], pose6, codes[index], fi["bg_color"],
                        tt.GOLDEN_DS, tt.GOLDEN_MAX_STEPS)
    tt.task_loss(orc, gt, tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    M = int(orc["mask"].sum())
    for k in ("torso_alpha_map", "torso_rgb_map", "rgb_map", "weights_sum"):
        report[f"b.{k}"] = rel(orc[k].detach().reshape(-1), res[k].detach().reshape(-1))
    for k in tt.TRAINABLE:
        report[f"b.grad.{k}"] = rel(p[k].grad, params[k].grad)
    report["b.grad.code"] = rel(codes.grad[tt.GOLDEN_INDEX], params["torso_individual_codes"].grad[tt.GOLDEN_INDEX])
    report["b.masked_pixels"] = M
    g.update({"b.rays_o": fi["rays_o"].numpy(), "b.rays_d": fi["rays_d"].numpy(), "b.cond": fi["cond"].numpy(), "b.bg_coords": fi["bg_coords"].numpy(),
              "b.bg_color": fi["bg_color"].numpy(), "b.gt": gt.numpy(), "b.cond_feat": cond_feat.reshape(-1).numpy()})
    for k in ("torso_alpha_map", "torso_rgb_map", "rgb_map", "weights_sum"):
        g[f"b.{k}"] = res[k].detach().numpy()
    store_grads(g, "b.grad", {k: params[k].grad for k in WEIGHTS}, params["torso_individual_codes"].grad[tt.GOLDEN_INDEX],
                params["torso_embedder.embeddings"].grad, offsets, idx)
    p64 = tt.torso_params(sc.state, torch.float64)
    codes64 = sc.state["torso_individual_codes"].double().clone().requires_grad_(True)
    o64 = tt.train_step(hpar, p64, hp, sc.state, fi["rays_o"], fi["rays_d"], cond_feat, ind, fi["bg_coords"], pose6, codes64[index], fi["bg_color"],
                        tt.GOLDEN_DS, tt.GOLDEN_MAX_STEPS)
    tt.task_loss(o64, gt, tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    store_grads(g, "b.grad64", {k: p64[k].grad for k in WEIGHTS}, codes64.grad[tt.GOLDEN_INDEX], p64["torso_embedder.embeddings"].grad, offsets, idx)
    for k in WEIGHTS:
        report[f"b.fp32_vs_fp64.{k}"] = rel(params[k].grad, p64[k].grad)
    report["b.fp32_vs_fp64.code"] = rel(params["torso_individual_codes"].grad[tt.GOLDEN_INDEX], codes64.grad[tt.GOLDEN_INDEX])
    g["table_sample_idx"] = idx
    os.chdir(cwd)

    print(f"(a) {tt.GOLDEN_M} points, {n_out} with shrink * x + dx outside [-1, 1];  (b) {M} of {N} pixels in the torso mask")
    for k, v in report.items():
        print(f"  {k}: {v if isinstance(v, int) else f'{v:.3e}'}")
    worst = max(v for k, v in report.items() if not isinstance(v, int) and "fp32_vs_fp64" not in k)
    print(f"WORST relative max|reference - oracle| = {worst:.3e}")
    if worst > 1e-5 or n_out == 0 or not 0 < M < N:
        return 1
    meta = dict(source="reference RADNeRFTorso.forward_torso and render() (training branch) + backward on CPU via oracle/ref_shim.py + "
                "oracle/ref_train_shim.py", density_scale=tt.GOLDEN_DS, index=tt.GOLDEN_INDEX, frame=tt.GOLDEN_FRAME, max_steps=tt.GOLDEN_MAX_STEPS,
                deform_gain=tt.DEFORM_GAIN, report=report, torch=torch.__version__)
    g["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(ROOT, "tests", "golden", "train_torso.npz")
    np.savez_compressed(path, **g)
    print(f"wrote tests/golden/train_torso.npz ({os.path.getsize(path) / 1024:.0f} KB)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
