"""oracle/make_torso_sr_train_golden.py -- pins the training torso-SR field against the reference's OWN RADNeRFTorsowithSR
(modules/radnerfs/radnerf_torso_sr.py) and its backward, and writes tests/golden/train_torso_sr.npz.

Runs only where the reference sources exist.  The reference's RADNeRFTorsowithSR is built from
egs/datasets/May/lm3d_radnerf_torso_sr.yaml, loads the synthetic state of oracle/torso_sr_train.golden_state() (deform output layer
scaled by DEFORM_GAIN) with strict=True, is put in .train() mode with on_train_torso_nerf() (the parameters RADNeRFTorsoSRTask
trains) and runs on the CPU through oracle/ref_shim.py plus oracle/ref_train_shim.py.  Three parts, each forward_torso at GOLDEN_M
seeded points (some where shrink * x + dx leaves [-1, 1]) for landmarks lm68_sequence(4)[GOLDEN_FRAME], then backward of a seeded
linear loss of alpha, color and dx:
  (a) torso_head_aware, code row torso_individual_codes[index] (index a [1] tensor, as the task passes it), per-point image and
      weights_sum;
  (b) the same with image=None (the encoder sees zeros);
  (c) torso_head_aware false and torso_individual_embedding_dim 0 (no code).
The same computations through oracle/torso_sr_train.py (the checker) are compared with it; the script fails if any output or gradient
differs by more than 1e-5 relative.  The inputs are not stored: tests regenerate them from the seeds (golden_points, golden_state).

Stored per part: the reference's outputs and fp32 gradients of every trainable parameter (the table at N_SAMPLE seeded entries and
its per-level L2 norms) and the same gradients from the checker with float64 dense layers.

Usage:  python -m oracle.make_torso_sr_train_golden
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ops, ref_shim, ref_train_shim  # noqa: E402
from oracle import torso_sr_train as tst  # noqa: E402

N_SAMPLE = 2048


def table_sample(n_entries):
    return np.sort(np.random.Generator(np.random.PCG64(23)).choice(n_entries, N_SAMPLE, replace=False)).astype(np.int64)


def level_norms(grad, offsets):
    off = offsets.tolist()
    return np.asarray([float(grad[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)], dtype=np.float64)


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def store(g, prefix, grads, offsets, idx):
    for k, v in grads.items():
        v = v.detach()
        if k == "torso_embedder.embeddings":
            g[f"{prefix}.table_sample"] = v[idx].numpy().astype(np.float32)
            g[f"{prefix}.table_level_norms"] = level_norms(v, offsets)
        else:
            g[f"{prefix}.{k}"] = v.numpy().astype(np.float32)


def main():
    cwd = os.getcwd()
    ops.build()
    set_hparams = ref_shim.install(ops)
    ref_train_shim.install_training(ops)
    from modules.radnerfs.radnerf_torso_sr import RADNeRFTorsowithSR
    lm68 = tst.golden_lm68()
    idx = None
    report, g = {}, {}
    for part, over in tst.PARTS.items():
        hp = tst.golden_hparams(part)
        hstr = ",".join(f"{k}={v}" for k, v in over.items())
        ref_hp = set_hparams("egs/datasets/May/lm3d_radnerf_torso_sr.yaml", hparams_str=hstr, print_hparams=False)
        for k in ("torso_shrink", "torso_individual_embedding_dim", "torso_head_aware", "grid_interpolation_type"):
            assert ref_hp[k] == hp[k], (part, k, ref_hp[k], hp[k])
        state = tst.golden_state(hp)
        model = RADNeRFTorsowithSR(ref_hp)
        model.load_state_dict(state, strict=True)
        model.train()
        model.on_train_torso_nerf()
        offsets = state["torso_embedder.offsets"]
        if idx is None:
            idx = table_sample(int(offsets[-1]))
        head_aware = bool(hp["torso_head_aware"])
        has_code = hp["torso_individual_embedding_dim"] > 0
        pts = tst.golden_points()
        image, ws = (pts["image"], pts["weights_sum"]) if part == "a" else (None, None)
        index = torch.tensor([tst.GOLDEN_INDEX])
        params = dict(model.named_parameters())
        model.zero_grad(set_to_none=True)
        c = model.torso_individual_codes[index] if has_code else None
        a, col, dx = model.forward_torso(pts["x"], torch.zeros(1, 6), c, image, ws, lm68=lm68)   # poses: read, unused
        tst.linear_loss(a, col, dx, pts).backward()
        names = tst.trainable(head_aware)
        ref_grads = {k: params[k].grad for k in names}
        if has_code:
            ref_grads["code"] = params["torso_individual_codes"].grad[tst.GOLDEN_INDEX]
        for k, v in params.items():     # on_train_torso_nerf: nothing else (sr_net, the head) receives a gradient
            if k not in names and k != "torso_individual_codes":
                assert v.grad is None, (part, k)

        def oracle(dtype):
            p = tst.torso_sr_params(state, head_aware, dtype)
            codes = state["torso_individual_codes"].to(dtype).clone().requires_grad_(True) if has_code else None
            trace = {}
            o = tst.torso_sr_forward(p, hp, pts["x"], lm68, codes[index] if has_code else None, image, ws, trace)
            tst.linear_loss(*o, pts).backward()
            gr = {k: p[k].grad for k in names}
            if has_code:
                gr["code"] = codes.grad[tst.GOLDEN_INDEX]
            return o, gr, trace

        (oa, oc, odx), og, trace = oracle(torch.float32)
        for k, (r, o) in {"alpha": (a, oa), "color": (col, oc), "deform": (dx, odx)}.items():
            report[f"{part}.{k}"] = rel(o.detach(), r.detach())
        for k in ref_grads:
            report[f"{part}.grad.{k}"] = rel(og[k], ref_grads[k])
        n_out = int((trace["x_pre_clamp"].abs() > 1).any(-1).sum())
        report[f"{part}.points_leaving"] = n_out
        _, og64, _ = oracle(torch.float64)
        for k in ref_grads:
            report[f"{part}.fp32_vs_fp64.{k}"] = rel(ref_grads[k], og64[k])
        g.update({f"{part}.alpha": a.detach().numpy(), f"{part}.color": col.detach().numpy(), f"{part}.deform": dx.detach().numpy()})
        store(g, f"{part}.grad", ref_grads, offsets, idx)
        store(g, f"{part}.grad64", og64, offsets, idx)
    g["table_sample_idx"] = idx
    os.chdir(cwd)

    for k, v in report.items():
        print(f"  {k}: {v if isinstance(v, int) else f'{v:.3e}'}")
    worst = max(v for k, v in report.items() if not isinstance(v, int) and "fp32_vs_fp64" not in k)
    print(f"WORST relative max|reference - oracle| = {worst:.3e}")
    if worst > 1e-5 or any(report[f"{p}.points_leaving"] == 0 for p in tst.PARTS):
        return 1
    meta = dict(source="reference RADNeRFTorsowithSR.forward_torso (on_train_torso_nerf, training mode) + backward on CPU via "
                "oracle/ref_shim.py + oracle/ref_train_shim.py", index=tst.GOLDEN_INDEX, frame=tst.GOLDEN_FRAME, M=tst.GOLDEN_M,
                deform_gain=tst.DEFORM_GAIN, parts=tst.PARTS, report=report, torch=torch.__version__)
    g["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(ROOT, "tests", "golden", "train_torso_sr.npz")
    np.savez_compressed(path, **g)
    print(f"wrote tests/golden/train_torso_sr.npz ({os.path.getsize(path) / 1024:.0f} KB)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
