"""oracle/make_grid_golden.py -- pins oracle/grid.py against the reference's own NeRFRenderer.update_extra_state and
mark_untrained_grid (modules/radnerfs/renderer.py:131-284) and writes tests/golden/grid_head32.npz, grid_head128.npz and
grid_untrained128.npz.

Runs only where /root/reference exists.  The reference's RADNeRF is built from egs/datasets/May/lm3d_radnerf.yaml (grid_size
overridden to 32 for the small case), loads genefaceplusplus_b200.scene.make_state with strict=True and runs on CPU through
oracle/ref_shim.py, with these substitutions for the duration of each call:
  * raymarching.morton3D / morton3D_dilation / packbits -> the C restatement (the wrappers force .cuda());
  * torch.rand_like -> the next cascade's slice of `noise` (scene.hashed_uniform, reproducible anywhere without an RNG);
  * random.randint -> the fixed conditioning index COND_INDEX;
  * Tensor.cuda -> identity (mark_untrained_grid moves its buffers to the GPU).

Usage:  python -m oracle.make_grid_golden
"""
import json
import os
import random
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from genefaceplusplus_b200.config import may_hparams, may_intrinsics  # noqa: E402
from oracle import grid as og  # noqa: E402
from oracle import ops, ref_shim  # noqa: E402
from oracle.render import OracleModel  # noqa: E402

DS = 8.0                 # density_scale of the refresh cases
DECAY = 0.95
COND_INDEX = 3
N_SAMPLE = 4096          # cells of the 128^3 grid whose raw / EMA values are stored
UNTRAINED_FRAMES = list(range(0, 100, 12))


def inputs(H):
    """Everything one refresh case needs; the tests rebuild it from here."""
    hp = may_hparams(grid_size=H)
    state = scn.make_state(torso=False, hparams=hp)
    C = 1
    conds = scn.cond_sequence(8)
    cond = scn.cond_window(conds, COND_INDEX, hp["smo_win_size"])
    noise = (scn.hashed_uniform(C * H ** 3 * 3, 311, 1.0) + 0.5).reshape(C, H, H, H, 3)
    grid0 = (scn.hashed_uniform(C * H ** 3, 312, 1.0) + 0.5).reshape(C, -1) * (2 * DS)
    grid0.view(-1)[::7] = -1.0             # untrained cells: the EMA must leave them at -1
    state["density_grid"] = grid0.clone()
    return dict(hp=hp, state=state, conds=conds, cond=cond, noise=noise, grid0=grid0)


def sample_cells(n_cells):
    return np.sort(np.random.Generator(np.random.PCG64(5)).choice(n_cells, N_SAMPLE, replace=False)).astype(np.int64)


def untrained_inputs():
    poses = torch.stack([scn.camera_pose(t) for t in UNTRAINED_FRAMES])
    return poses, tuple(float(v) for v in may_intrinsics(512, 512))


class _Patched:
    """Context: the substitutions listed in the module docstring."""

    def __init__(self, rm, noise=None):
        self.rm, self.noise, self.calls = rm, noise, 0

    def __enter__(self):
        rm = self.rm
        self.saved = (rm.morton3D, rm.morton3D_dilation, rm.packbits, torch.rand_like, random.randint, torch.Tensor.cuda)
        rm.morton3D = ops.morton3D
        rm.morton3D_dilation = ops.morton3D_dilation
        rm.packbits = lambda grid, thresh, bitfield=None: ops.packbits(grid, thresh)

        def rand_like(t, *a, **k):
            out = self.noise[self.calls].reshape(t.shape).clone()
            self.calls += 1
            return out
        torch.rand_like = rand_like
        random.randint = lambda a, b: COND_INDEX
        torch.Tensor.cuda = lambda self_, *a, **k: self_
        return self

    def __exit__(self, *exc):
        rm = self.rm
        rm.morton3D, rm.morton3D_dilation, rm.packbits, torch.rand_like, random.randint, torch.Tensor.cuda = self.saved


def main():
    cwd = os.getcwd()
    ops.build()
    set_hparams = ref_shim.install(ops)
    import modules.radnerfs.raymarching as rm
    from modules.radnerfs.radnerf import RADNeRF
    out_dir = os.path.join(ROOT, "tests", "golden")
    files, worst, report = {}, 0.0, {}
    for H in (32, 128):
        inp = inputs(H)
        ref_hp = set_hparams("egs/datasets/May/lm3d_radnerf.yaml", hparams_str=f"grid_size={H}", print_hparams=False)
        assert ref_hp["grid_size"] == H and ref_hp["smo_win_size"] == inp["hp"]["smo_win_size"]
        with torch.no_grad():
            model = RADNeRF(ref_hp).eval()
        model.load_state_dict(inp["state"], strict=True)
        model.density_scale = DS
        model.conds = inp["conds"]
        t0 = time.time()
        with torch.no_grad(), _Patched(rm, inp["noise"]) as p:
            # the raw grid is a local of update_extra_state: recover it by wrapping the dilation it is passed to
            seen = {}
            dil = rm.morton3D_dilation
            rm.morton3D_dilation = lambda g: (seen.__setitem__("tmp", g.clone()), dil(g))[1]
            model.update_extra_state(decay=DECAY, S=128)
            assert p.calls == 1, p.calls
        t1 = time.time()
        orc = OracleModel(inp["state"], inp["hp"], torso=False)
        orc.density_scale = DS
        # the refresh is pinned on the reference's own conditioning vector (stored in the golden); the oracle's cal_cond_feat
        # agrees with it to ~1 ulp, which exp() of the sigma logit turns into a few 1e-6 relative (printed)
        cf = model.cal_cond_feat(inp["cond"]).detach()
        d_cond = (orc.cal_cond_feat(inp["cond"]).reshape(-1) - cf.reshape(-1)).abs().max().item()
        tmp, grid, mean, bits = og.update_extra_state(orc, cf, inp["noise"], inp["grid0"], DECAY, float(ref_hp["density_thresh"]))
        t2 = time.time()
        ref_tmp, ref_grid = seen["tmp"], model.density_grid.clone()
        ref_bits, ref_mean = model.density_bitfield.clone(), float(model.mean_density)
        d_tmp = ((ref_tmp - tmp).abs() / ref_tmp.abs().clamp(min=1)).max().item()
        d_grid = ((ref_grid - grid).abs() / ref_grid.abs().clamp(min=1)).max().item()
        d_mean = abs(ref_mean - mean) / abs(ref_mean)
        n_bits = int((ref_bits != bits).sum())
        occ = float(np.unpackbits(ref_bits.numpy()).mean())
        print(f"  head grid {H}^3: cal_cond_feat max|ref-oracle| {d_cond:.3e} (not gated); rel max|ref-oracle| raw {d_tmp:.3e}, EMA {d_grid:.3e}, mean {d_mean:.3e} (mean {ref_mean:.6f}); "
              f"bitfield bytes differing {n_bits}; occupancy {occ:.3f}; ref {t1-t0:.1f}s oracle {t2-t1:.1f}s")
        worst = max(worst, d_tmp, d_grid, d_mean, float(n_bits))
        report[f"head{H}"] = dict(cond_feat=d_cond, raw=d_tmp, ema=d_grid, mean=d_mean, bitfield_bytes=n_bits, occupancy=occ)
        g = {"mean": np.asarray([ref_mean], dtype=np.float64), "bitfield": ref_bits.numpy(), "cond_feat": cf.reshape(-1).numpy().astype(np.float32)}
        if H == 32:
            g.update(raw=ref_tmp.numpy().astype(np.float32), ema=ref_grid.numpy().astype(np.float32))
        else:
            idx = sample_cells(ref_tmp.numel())
            g.update(cells=idx, raw=ref_tmp.reshape(-1)[idx].numpy().astype(np.float32), ema=ref_grid.reshape(-1)[idx].numpy().astype(np.float32))
        files[f"grid_head{H}.npz"] = g
        if H == 128:
            poses, intr = untrained_inputs()
            model.density_grid.zero_()
            with torch.no_grad(), _Patched(rm):
                model.mark_untrained_grid(poses, intr, S=64)
            ref_mark = model.density_grid.clone()
            mine = og.mark_untrained_grid(orc, torch.zeros_like(ref_mark), poses, intr, S=64)
            n_flip = int(((ref_mark == -1) != (mine == -1)).sum())
            n_untrained = int((ref_mark == -1).sum())
            print(f"  mark_untrained_grid {H}^3, {len(UNTRAINED_FRAMES)} poses: {n_untrained} of {ref_mark.numel()} cells untrained; "
                  f"cells differing from the oracle {n_flip}")
            worst = max(worst, float(n_flip))
            report["untrained128"] = dict(untrained=n_untrained, differing=n_flip)
            files["grid_untrained128.npz"] = {"untrained_bits": np.packbits((ref_mark.reshape(-1) == -1).numpy().astype(np.uint8)),
                                              "n_untrained": np.asarray([n_untrained])}
    os.chdir(cwd)
    print(f"WORST relative max|reference - oracle| (or count of differing cells/bytes) = {worst:.3e}")
    if worst > 2e-6:
        return 1
    for name, g in files.items():
        meta = dict(source="reference NeRFRenderer.update_extra_state / mark_untrained_grid on CPU via oracle/ref_shim.py",
                    density_scale=DS, decay=DECAY, cond_index=COND_INDEX, untrained_frames=UNTRAINED_FRAMES, report=report,
                    torch=torch.__version__)
        g["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(out_dir, name), **g)
        print(f"wrote tests/golden/{name} ({os.path.getsize(os.path.join(out_dir, name)) / 1024:.0f} KB)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
