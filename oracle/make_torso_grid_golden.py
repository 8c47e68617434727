"""oracle/make_torso_grid_golden.py -- pins oracle/torso_grid.py against the reference's own RADNeRFTorso.update_extra_state
(modules/radnerfs/radnerf_torso.py:201-242) and RADNeRFTorsowithSR.update_extra_state (radnerf_torso_sr.py:246-288) and writes
tests/golden/torso_grid128.npz, torso_grid32.npz and torso_sr_grid128.npz.

Runs only where /root/reference exists.  The reference's models are built from egs/datasets/May/lm3d_radnerf_torso.yaml (grid_size
overridden to 32 for the small case) and lm3d_radnerf_torso_sr.yaml (head-aware), load genefaceplusplus_b200.scene.make_state /
make_torso_sr_state with strict=True and run on CPU through oracle/ref_shim.py, with these substitutions for the duration of each
call:
  * random.randint -> the fixed training-pose index POSE_INDEX;
  * torch.rand_like -> `noise` (scene.hashed_uniform, reproducible anywhere without an RNG; one chunk since S >= grid_size);
  * F.max_pool2d wrapped, so that the raw (pre-dilation) grid, a local of update_extra_state, is recovered;
  * the module's convert_poses wrapped, so that the pose the reference conditions on is stored;
  * model.poses / model.lm68s <- scene.camera_pose / scene.lm68_sequence (the training task sets them in the reference).
The starting grid is hashed in [0, GRID_AMP): grid * decay beats the dilated alphas on a sizeable share of the cells (printed), so
both sides of the EMA's max are exercised.

Usage:  python -m oracle.make_torso_grid_golden
"""
import json
import os
import random
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.config import may_hparams  # noqa: E402
from oracle import ops, ref_shim  # noqa: E402
from oracle import torso_grid as otg  # noqa: E402
from oracle.render import OracleModel  # noqa: E402

DECAY = 0.95
POSE_INDEX = 5
N_POSES = 8
GRID_AMP = 1.6
NOISE_SALT, GRID_SALT = 411, 412
SR_OVERRIDES = dict(with_sr=True, torso_head_aware=True, add_eye_blink_cond=True, eye_blink_dim=4, smo_win_size=3)
CASES = {"torso_grid128.npz": ("torso", 128), "torso_grid32.npz": ("torso", 32), "torso_sr_grid128.npz": ("torso_sr", 128)}


def inputs(kind, H):
    """Everything one refresh case needs; the tests rebuild it from here."""
    if kind == "torso_sr":
        hp = may_hparams(grid_size=H, **SR_OVERRIDES)
        state = scn.make_torso_sr_state(hp)
    else:
        hp = may_hparams(grid_size=H)
        state = scn.make_state(torso=True, hparams=hp)
    noise = (scn.hashed_uniform(H * H * 2, NOISE_SALT, 1.0) + 0.5).reshape(H, H, 2)
    grid0 = (scn.hashed_uniform(H * H, GRID_SALT, 1.0) + 0.5) * GRID_AMP
    state["density_grid_torso"] = grid0.clone()
    poses = torch.stack([scn.camera_pose(t) for t in range(N_POSES)])
    lm68s = scn.lm68_sequence(N_POSES)
    code = state["torso_individual_codes"][POSE_INDEX].clone()
    return dict(hp=hp, state=state, noise=noise, grid0=grid0, poses=poses, lm68s=lm68s, code=code)


class _Patched:
    """Context: the substitutions listed in the module docstring."""

    def __init__(self, mod, noise):
        self.mod, self.noise, self.calls, self.seen = mod, noise, 0, {}

    def __enter__(self):
        self.saved = (torch.rand_like, random.randint, F.max_pool2d, self.mod.convert_poses)

        def rand_like(t, *a, **k):
            self.calls += 1
            return self.noise.reshape(t.shape).clone()
        torch.rand_like = rand_like
        random.randint = lambda a, b: POSE_INDEX
        pool, conv = self.saved[2], self.saved[3]
        F.max_pool2d = lambda g, *a, **k: (self.seen.__setitem__("tmp", g.reshape(-1).clone()), pool(g, *a, **k))[1]
        self.mod.convert_poses = lambda p: (lambda out: (self.seen.__setitem__("pose6", out.reshape(-1).clone()), out)[1])(conv(p))
        return self

    def __exit__(self, *exc):
        torch.rand_like, random.randint, F.max_pool2d, self.mod.convert_poses = self.saved


def main():
    cwd = os.getcwd()
    ops.build()
    set_hparams = ref_shim.install(ops)
    import modules.radnerfs.radnerf_torso as mod_torso
    import modules.radnerfs.radnerf_torso_sr as mod_torso_sr
    out_dir = os.path.join(ROOT, "tests", "golden")
    files, worst, report = {}, 0.0, {}
    for name, (kind, H) in CASES.items():
        inp = inputs(kind, H)
        if kind == "torso_sr":
            mod, cls, yaml = mod_torso_sr, mod_torso_sr.RADNeRFTorsowithSR, "egs/datasets/May/lm3d_radnerf_torso_sr.yaml"
        else:
            mod, cls, yaml = mod_torso, mod_torso.RADNeRFTorso, "egs/datasets/May/lm3d_radnerf_torso.yaml"
        ref_hp = set_hparams(yaml, hparams_str=f"grid_size={H}", print_hparams=False)
        assert ref_hp["grid_size"] == H and bool(ref_hp["torso_head_aware"]) == (kind == "torso_sr")
        with torch.no_grad():
            model = cls(ref_hp).eval()
        model.load_state_dict(inp["state"], strict=True)
        model.poses = inp["poses"]
        model.lm68s = inp["lm68s"]
        t0 = time.time()
        with torch.no_grad(), _Patched(mod, inp["noise"]) as p:
            model.update_extra_state(decay=DECAY, S=128)
            assert p.calls == 1, p.calls
        t1 = time.time()
        ref_tmp, ref_grid, ref_mean, pose6 = p.seen["tmp"], model.density_grid_torso.clone(), float(model.mean_density_torso), p.seen["pose6"]
        orc = OracleModel(inp["state"], inp["hp"], torso=True)
        lm68 = inp["lm68s"][POSE_INDEX] if kind == "torso_sr" else None
        tmp, grid, mean = otg.update_extra_state(orc, inp["noise"], inp["grid0"], DECAY, pose6=pose6, code=inp["code"], lm68=lm68)
        t2 = time.time()
        d_tmp = (ref_tmp - tmp).abs().max().item()
        d_grid = (ref_grid - grid).abs().max().item()
        d_mean = abs(ref_mean - mean) / abs(ref_mean)
        dil = F.max_pool2d(ref_tmp.view(1, 1, H, H), 5, 1, 2).reshape(-1)
        ema_share = float((inp["grid0"] * DECAY > dil).float().mean())
        print(f"  {name}: max|ref-oracle| raw {d_tmp:.3e}, EMA {d_grid:.3e}, rel mean {d_mean:.3e} (mean {ref_mean:.6f}); alpha range "
              f"[{ref_tmp.min().item():.3f}, {ref_tmp.max().item():.3f}]; cells where grid*decay wins {ema_share:.3f}; "
              f"ref {t1-t0:.1f}s oracle {t2-t1:.1f}s")
        worst = max(worst, d_tmp, d_grid, d_mean)
        report[name] = dict(raw=d_tmp, ema=d_grid, mean=d_mean, ema_share=ema_share)
        g = {"raw": ref_tmp.numpy().astype(np.float32), "ema": ref_grid.numpy().astype(np.float32),
             "mean": np.asarray([ref_mean], dtype=np.float64), "pose_index": np.asarray([POSE_INDEX]),
             "code": inp["code"].numpy().astype(np.float32)}
        if kind == "torso_sr":
            g["lm68"] = lm68.numpy().astype(np.float32)
        else:
            g["pose6"] = pose6.numpy().astype(np.float32)
        files[name] = g
    os.chdir(cwd)
    print(f"WORST max|reference - oracle| = {worst:.3e}")
    if worst > 2e-6:
        return 1
    for name, g in files.items():
        meta = dict(source="reference RADNeRFTorso / RADNeRFTorsowithSR.update_extra_state on CPU via oracle/ref_shim.py", decay=DECAY,
                    pose_index=POSE_INDEX, n_poses=N_POSES, grid_amp=GRID_AMP, noise_salt=NOISE_SALT, grid_salt=GRID_SALT,
                    report=report[name], torch=torch.__version__)
        g["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(out_dir, name), **g)
        print(f"wrote tests/golden/{name} ({os.path.getsize(os.path.join(out_dir, name)) / 1024:.0f} KB)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
