"""oracle/make_train_golden.py -- pins the training field and the training branch of render() against the reference's OWN
RADNeRF.render (modules/radnerfs/renderer.py:286-339, 385-398) and its backward, and writes tests/golden/train_head.npz.

Runs only where /root/reference exists.  The reference's RADNeRF is built from egs/datasets/May/lm3d_radnerf.yaml, loads the synthetic
May scene (genefaceplusplus_b200.scene.Scene(H=32, W=32), frame 1: 1024 rays) with strict=True and runs on the CPU through
oracle/ref_shim.py plus oracle/ref_train_shim.py (its training wrappers on the C restatement), in .train() mode with perturb=False,
max_steps 16, density_scale 8 and individual code row INDEX.  The loss is a fixed, seeded linear functional of rgb_map, weights_sum and
ambient.  The same step through oracle/field_train.render_train (the checker) is compared with it and the difference printed.

Stored: the inputs and loss coefficients; the reference's outputs and `position`; the gradients of the eight MLP weights (full), of
individual_embeddings[INDEX] and of every cond_prenet / cond_att_net parameter; for both tables, the gradient at N_SAMPLE seeded
entries and its per-level L2 norms.

Usage:  python -m oracle.make_train_golden
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from oracle import field_train as ft  # noqa: E402
from oracle import ops, ref_shim, ref_train_shim  # noqa: E402

DS = 8.0
INDEX = 2
FRAME = 1
MAX_STEPS = 16
N_SAMPLE = 2048
TABLES = ("position_embedder", "ambient_embedder")


def scene():
    return scn.Scene(H=32, W=32, T=4, torso=False, density_scale=DS)


def coefficients(N):
    g = torch.Generator().manual_seed(1234)
    return torch.randn(N, 3, generator=g), torch.randn(N, generator=g), torch.randn(N, generator=g)


def loss_of(res, coef):
    return (res["rgb_map"].reshape(-1, 3) * coef[0]).sum() + (res["weights_sum"] * coef[1]).sum() + (res["ambient"] * coef[2]).sum()


def table_sample(n_entries, name):
    return np.sort(np.random.Generator(np.random.PCG64(17 + len(name))).choice(n_entries, N_SAMPLE, replace=False)).astype(np.int64)


def level_norms(grad, offsets):
    off = offsets.tolist()
    return np.asarray([float(grad[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)], dtype=np.float64)


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def main():
    cwd = os.getcwd()
    ops.build()
    set_hparams = ref_shim.install(ops)
    ref_train_shim.install_training(ops)
    from modules.radnerfs.radnerf import RADNeRF
    sc = scene()
    ref_hp = set_hparams("egs/datasets/May/lm3d_radnerf.yaml", hparams_str="", print_hparams=False)
    for k in ("grid_size", "bound", "desired_resolution", "ambient_coord_dim", "individual_embedding_dim", "smo_win_size", "min_near"):
        assert ref_hp[k] == sc.hparams[k], (k, ref_hp[k], sc.hparams[k])
    model = RADNeRF(ref_hp)
    model.load_state_dict(sc.state, strict=True)
    model.density_scale = DS
    model.train()
    fi = sc.frame_inputs(FRAME)
    N = fi["rays_o"].numel() // 3
    coef = coefficients(N)
    res = model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=INDEX, dt_gamma=0, bg_color=fi["bg_color"],
                       perturb=False, force_all_rays=False, max_steps=MAX_STEPS)
    loss_of(res, coef).backward()
    params = dict(model.named_parameters())
    with torch.no_grad():
        cond_feat = model.cal_cond_feat(fi["cond"]).detach()

    # the checker on the same step
    p = ft.field_params(sc.state)
    emb = sc.state["individual_embeddings"].clone().requires_grad_(True)
    orc = ft.render_train(p, sc.hparams, sc.state, fi["rays_o"], fi["rays_d"], cond_feat, emb[INDEX], fi["bg_color"], DS, MAX_STEPS)
    loss_of(orc, coef).backward()
    report = {}
    for k in ("rgb_map", "weights_sum", "ambient", "depth_map"):
        report[k] = rel(orc[k].detach(), res[k].detach())
    report["position_equal"] = bool(torch.equal(orc["position"], res["position"]))
    for k in ft.TRAINABLE:
        report[k] = rel(p[k].grad, params[k].grad)
    report["individual_embeddings"] = rel(emb.grad[INDEX], params["individual_embeddings"].grad[INDEX])
    os.chdir(cwd)
    print(f"training step: {res['position'].shape[0]} samples of {N} rays")
    for k, v in report.items():
        print(f"  reference vs oracle {k}: {v if isinstance(v, bool) else f'{v:.3e}'}")
    worst = max(v for v in report.values() if not isinstance(v, bool))
    print(f"WORST relative max|reference - oracle| = {worst:.3e}")
    if worst > 1e-4 or not report["position_equal"]:
        return 1

    g = {"rays_o": fi["rays_o"].numpy(), "rays_d": fi["rays_d"].numpy(), "cond": fi["cond"].numpy(), "bg_color": fi["bg_color"].numpy(),
         "coef_rgb": coef[0].numpy(), "coef_ws": coef[1].numpy(), "coef_amb": coef[2].numpy(), "cond_feat": cond_feat.reshape(-1).numpy()}
    for k in ("rgb_map", "weights_sum", "ambient", "depth_map", "position"):
        g[k] = res[k].detach().numpy()
    for k in ft.TRAINABLE[:8]:
        g["grad." + k] = params[k].grad.numpy()
    g["grad.individual_code"] = params["individual_embeddings"].grad[INDEX].numpy()
    # the same step with the checker's dense layers in float64: what the reference's fp32 gradients approximate (their own rounding
    # is large where a weight gradient is a column sum that cancels, e.g. ambient_net.0's conditioning columns)
    p64 = ft.field_params(sc.state, torch.float64)
    emb64 = sc.state["individual_embeddings"].double().clone().requires_grad_(True)
    o64 = ft.render_train(p64, sc.hparams, sc.state, fi["rays_o"], fi["rays_d"], cond_feat.double(), emb64[INDEX], fi["bg_color"], DS, MAX_STEPS)
    loss_of(o64, tuple(c.double() for c in coef)).backward()
    for k in ft.TRAINABLE[:8]:
        g["grad64." + k] = p64[k].grad.numpy().astype(np.float32)   # stored in fp32: its rounding (6e-8) is far below what it measures
        report["fp32_vs_fp64." + k] = rel(params[k].grad, p64[k].grad)
    g["grad64.individual_code"] = emb64.grad[INDEX].numpy().astype(np.float32)
    print("  reference fp32 vs float64 dense layers: " + ", ".join(f"{k[13:]} {v:.2e}" for k, v in report.items() if k.startswith("fp32_vs")))
    for k, v in params.items():
        if k.startswith(("cond_prenet.", "cond_att_net.")):
            g["grad." + k] = v.grad.numpy()
    for t in TABLES:
        gr = params[f"{t}.embeddings"].grad
        idx = table_sample(gr.shape[0], t)
        g[f"{t}.sample_idx"] = idx
        g[f"{t}.sample_grad"] = gr[idx].numpy()
        g[f"{t}.level_norms"] = level_norms(gr, sc.state[f"{t}.offsets"])
    meta = dict(source="reference RADNeRF.render (training branch) + backward on CPU via oracle/ref_shim.py + oracle/ref_train_shim.py",
                density_scale=DS, index=INDEX, frame=FRAME, max_steps=MAX_STEPS, report=report, torch=torch.__version__)
    g["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(ROOT, "tests", "golden", "train_head.npz")
    np.savez_compressed(path, **g)
    print(f"wrote tests/golden/train_head.npz ({os.path.getsize(path) / 1024:.0f} KB)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
