"""oracle/validate_against_reference.py -- pins the oracle against the reference's OWN Python.

Runs only where /root/reference exists (this container; never on the GPU box).  For each case it
  1. builds the reference's RADNeRF / RADNeRFTorso from the May yaml chain (oracle/ref_shim.py),
  2. load_state_dict(strict=True)s the synthetic state from genefaceplusplus_b200.scene
     (this also pins the state_dict key/shape contract, SURVEY.md 8(a) a16),
  3. calls the reference's unmodified `render()` on CPU with the native ops served by the C
     restatement, and
  4. compares with oracle.render.OracleModel.render on the same inputs.
Both sides share the native-op restatement, so (3) vs (4) pins the *host* logic the oracle restates
(round loop, MLP wiring, cond nets, torso composite); the native ops themselves are pinned on the
GPU against the reference's own CUDA kernels (tests/test_gpu_ref_pin.py).

Usage:  python -m oracle.validate_against_reference [--size 64] [--write-golden]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from oracle import ops, ref_shim  # noqa: E402
from oracle.render import OracleModel  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# (name, torso, H=W, max_steps, density_scale, frames)
CASES = [
    ("head64_ms8_ds1", False, 64, 8, 1.0, (0, 1, 2, 3)),     # BASELINE config 1 (plumbing case)
    ("head64_ms16_ds8", False, 64, 16, 8.0, (0, 7)),
    ("torso64_ms16_ds1", True, 64, 16, 1.0, (0, 3)),
    ("torso48_ms16_ds64", True, 48, 16, 64.0, (5,)),
]


def run_case(set_hparams, name, torso, size, max_steps, density_scale, frames, write_golden):
    cwd = os.getcwd()
    model, hp = ref_shim.build_reference_model(set_hparams, torso=torso)
    sc = scn.Scene(H=size, W=size, T=8, torso=torso, max_steps=max_steps, density_scale=density_scale)
    missing = model.load_state_dict(sc.state, strict=True)
    model.density_scale = density_scale
    orc = OracleModel(sc.state, sc.hparams)
    orc.density_scale = density_scale
    out = {}
    worst = 0.0
    for t in frames:
        fi = sc.frame_inputs(t)
        kw = dict(hp)
        kw["max_steps"] = max_steps
        t0 = time.time()
        with torch.no_grad():
            ref = model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=t, staged=False,
                               bg_color=fi["bg_color"], perturb=False, force_all_rays=False, T_thresh=sc.T_thresh, **kw)
        t1 = time.time()
        mine = orc.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=t,
                          bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **{**sc.hparams})
        t2 = time.time()
        keys = ["rgb_map", "depth_map"] + (["torso_alpha_map", "torso_rgb_map", "deform"] if torso else [])
        for k in keys:
            d = (ref[k].float() - mine[k].float()).abs().max().item()
            worst = max(worst, d)
            print(f"  {name} frame {t}: {k:16s} max|ref-oracle| = {d:.3e}")
        st = mine["stats"]
        print(f"  {name} frame {t}: S={st['S']} N={st['N']} P={st['P']} schedule={st['schedule']} B={st['B_total']}  (ref {t1-t0:.1f}s, oracle {t2-t1:.1f}s)")
        out[f"f{t}_rgb_map"] = ref["rgb_map"].numpy().astype(np.float32)
        out[f"f{t}_depth_map"] = ref["depth_map"].numpy().astype(np.float32)
        out[f"f{t}_weights_sum"] = mine["weights_sum"].numpy().astype(np.float32)
        out[f"f{t}_knife"] = mine["knife"].numpy().astype(np.float32)
        if torso:
            out[f"f{t}_torso_alpha_map"] = ref["torso_alpha_map"].numpy().astype(np.float32)
            out[f"f{t}_torso_rgb_map"] = ref["torso_rgb_map"].numpy().astype(np.float32)
        out[f"f{t}_stats"] = np.frombuffer(json.dumps(st).encode(), dtype=np.uint8)
    if write_golden:
        meta = dict(name=name, torso=torso, size=size, max_steps=max_steps, density_scale=density_scale, frames=list(frames),
                    T_thresh=sc.T_thresh, source="reference RADNeRF(.Torso).render on CPU via oracle/ref_shim.py",
                    torch=torch.__version__, numpy=np.__version__)
        out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        os.makedirs(GOLDEN_DIR, exist_ok=True)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"{name}.npz"), **out)
    os.chdir(cwd)
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write-golden", action="store_true")
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    ops.build()
    set_hparams = ref_shim.install(ops)
    worst = 0.0
    for case in CASES:
        if args.only and args.only not in case[0]:
            continue
        print(f"[case] {case[0]}")
        worst = max(worst, run_case(set_hparams, *case, write_golden=args.write_golden))
    print(f"WORST max|reference - oracle| over all cases/keys: {worst:.3e}")
    return 0 if worst <= 1e-6 else 1


if __name__ == "__main__":
    sys.exit(main())
