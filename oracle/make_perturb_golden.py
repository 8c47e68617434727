"""oracle/make_perturb_golden.py -- pins oracle/perturb.py against the reference's own render(perturb=True) in eval mode.

Runs only where the reference tree exists.  The reference's validation_step calls run_model(sample, infer=False) with the model in
eval mode under no_grad, i.e. render(..., perturb=True, force_all_rays=False) (tasks/radnerfs/radnerf.py:127 and the torso / SR
tasks).  For each case this
  1. builds the reference's RADNeRF / RADNeRFTorso from the May yaml chain (oracle/ref_shim.py) and loads the synthetic state,
  2. seeds torch and calls its unmodified render(perturb=True) on CPU, with the reference's march_rays wrapper restated by
     oracle.perturb.march_rays (the perturb branch draws torch.rand(n_alive), raymarching.py:388-390) and the draw recorded,
  3. renders the oracle with the same seed (it must draw the same vector) and with the recorded vector passed explicitly,
and writes tests/golden/perturb_<case>.npz: the draw, the reference's outputs, and the oracle's B / S / P / knife margins.

Usage:  python -m oracle.make_perturb_golden
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
from oracle import ops, perturb, ref_shim  # noqa: E402
from oracle.render import OracleModel  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# (name, torso, H=W, max_steps, density_scale, frame, seed); dt_gamma is the May value 1/256 and max_steps 16, so rays outlive the
# first max_steps samples and the fused renderer's pass 2 runs
CASES = [
    ("perturb_head64_ds16", False, 64, 16, 16.0, 3, 11),
    ("perturb_torso48_ds8", True, 48, 16, 8.0, 5, 12),
]


def run_case(set_hparams, rm_modules, name, torso, size, max_steps, density_scale, frame, seed):
    model, hp = ref_shim.build_reference_model(set_hparams, torso=torso)
    sc = scn.Scene(H=size, W=size, T=8, torso=torso, max_steps=max_steps, density_scale=density_scale)
    model.load_state_dict(sc.state, strict=True)
    model.density_scale = density_scale
    fi = sc.frame_inputs(frame)
    kw = dict(hp)
    kw["max_steps"] = max_steps
    assert kw["dt_gamma"] == sc.hparams["dt_gamma"]

    draws = []

    def recording_march_rays(*args, **kwargs):
        before = torch.get_rng_state()
        out = perturb.march_rays(*args, **kwargs)
        if not torch.equal(before, torch.get_rng_state()):
            # replay the draw the wrapper just made from the saved state: the recorded vector is the reference's own
            after = torch.get_rng_state()
            torch.set_rng_state(before)
            draws.append(torch.rand(args[0], dtype=torch.float32))
            assert torch.equal(torch.get_rng_state(), after)
        return out

    for target in rm_modules:
        target.march_rays = recording_march_rays
    torch.manual_seed(seed)
    with torch.no_grad():
        ref = model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=frame, staged=False,
                           bg_color=fi["bg_color"], perturb=True, force_all_rays=False, T_thresh=sc.T_thresh, **kw)
    for target in rm_modules:
        target.march_rays = ops.march_rays
    assert len(draws) == 1 and draws[0].numel() == sc.H * sc.W, [d.numel() for d in draws]
    noises = draws[0]

    orc = OracleModel(sc.state, sc.hparams)
    orc.density_scale = density_scale
    torch.manual_seed(seed)
    seeded = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=frame,
                            bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **sc.hparams)
    assert torch.equal(seeded["noises"], noises), "the oracle must draw the reference's vector from the same seed"
    mine = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=frame,
                          bg_color=fi["bg_color"], T_thresh=sc.T_thresh, noises=noises, **sc.hparams)
    plain = orc.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=frame,
                       bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **sc.hparams)
    worst = 0.0
    keys = ["rgb_map", "depth_map"] + (["torso_alpha_map", "torso_rgb_map", "deform"] if torso else [])
    for k in keys:
        d = (ref[k].float() - mine[k].float()).abs().max().item()
        ds = (ref[k].float() - seeded[k].float()).abs().max().item()
        worst = max(worst, d, ds)
        print(f"  {name}: {k:16s} max|ref-oracle| = {d:.3e} (seeded draw {ds:.3e})")
    st, stp = mine["stats"], plain["stats"]
    dp = (ref["rgb_map"].float() - plain["rgb_map"].float()).abs().max().item()
    print(f"  {name}: S={st['S']} N={st['N']} P={st['P']} B={st['B_total']} schedule={st['schedule']}")
    print(f"  {name}: perturb=False for comparison: S={stp['S']} B={stp['B_total']}; max|rgb(perturb) - rgb(no perturb)| = {dp:.3e}")
    out = {"noises": noises.numpy().astype(np.float32),
           "rgb_map": ref["rgb_map"].numpy().astype(np.float32), "depth_map": ref["depth_map"].numpy().astype(np.float32),
           "weights_sum": mine["weights_sum"].numpy().astype(np.float32), "knife": mine["knife"].numpy().astype(np.float32)}
    if torso:
        out["torso_alpha_map"] = ref["torso_alpha_map"].numpy().astype(np.float32)
        out["torso_rgb_map"] = ref["torso_rgb_map"].numpy().astype(np.float32)
    meta = dict(name=name, torso=torso, size=size, max_steps=max_steps, density_scale=density_scale, frame=frame, seed=seed,
                T_thresh=sc.T_thresh, dt_gamma=kw["dt_gamma"], stats=st,
                source="reference RADNeRF(.Torso).render(perturb=True) in eval mode on CPU via oracle/ref_shim.py + oracle/perturb.py",
                torch=torch.__version__, numpy=np.__version__)
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    return worst, out


def main():
    cwd = os.getcwd()
    ops.build()
    set_hparams = ref_shim.install(ops)
    import modules.radnerfs.raymarching as rm  # noqa: E402
    import modules.radnerfs.raymarching.raymarching as rm_inner  # noqa: E402
    worst, outs = 0.0, {}
    for case in CASES:
        print(f"[case] {case[0]}")
        w, outs[case[0]] = run_case(set_hparams, (rm, rm_inner), *case)
        worst = max(worst, w)
    os.chdir(cwd)
    print(f"WORST max|reference - oracle| over all cases/keys: {worst:.3e}")
    if worst > 1e-6:
        return 1
    for name, out in outs.items():
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"{name}.npz"), **out)
        print(f"wrote tests/golden/{name}.npz")
    return 0


if __name__ == "__main__":
    sys.exit(main())
