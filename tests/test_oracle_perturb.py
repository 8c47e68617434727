"""perturb=True in the inference branch of render(), on the CPU oracle (oracle/perturb.py).

  * the oracle reproduces the reference's own render(perturb=True) (tests/golden/perturb_*.npz, oracle/make_perturb_golden.py);
  * the round-schedule lemma (SURVEY.md H1) still holds with jittered starts: the multi-round image, B and S equal those of
    ONE round of n_step = B marched from near + clamp(near*dt_gamma, dt_min, dt_max) * noise -- which is what lets the fused
    renderer jitter only where k_ray_setup starts a ray;
  * all-zero noise is perturb=False."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "perturb_*.npz")))


def _oracle(sc, ds):
    from oracle.render import OracleModel
    orc = OracleModel(sc.state, sc.hparams)
    orc.density_scale = ds
    return orc


def test_goldens_exist_and_stay_out_of_the_plain_render_goldens():
    import re
    names = [os.path.basename(p) for p in GOLDEN]
    assert any(n.startswith("perturb_head") for n in names) and any(n.startswith("perturb_torso") for n in names)
    assert not any(re.match(r"(head|torso)\d+_ms", n) for n in names)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_matches_reference_golden(oracle_ops, path):
    from oracle import perturb
    z = np.load(path)
    m = json.loads(bytes(z["meta"]).decode())
    sc = scn.Scene(H=m["size"], W=m["size"], T=8, torso=m["torso"], max_steps=m["max_steps"], density_scale=m["density_scale"])
    fi = sc.frame_inputs(m["frame"])
    noises = torch.from_numpy(z["noises"])
    orc = _oracle(sc, m["density_scale"])
    kw = dict(index=m["frame"], bg_color=fi["bg_color"], T_thresh=m["T_thresh"], **sc.hparams)
    res = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], noises=noises, **kw)
    worst = 0.0
    for k in ("rgb_map", "depth_map") + (("torso_alpha_map", "torso_rgb_map") if m["torso"] else ()):
        worst = max(worst, (res[k] - torch.from_numpy(z[k])).abs().max().item())
    print(f"[{m['name']}] max|oracle - reference| = {worst:.3e}")
    assert worst <= 1e-6
    st = res["stats"]
    assert (st["S"], st["B_total"], st["P"], st["schedule"]) == (m["stats"]["S"], m["stats"]["B_total"], m["stats"]["P"],
                                                                 [tuple(s) for s in m["stats"]["schedule"]])
    assert torch.equal(res["weights_sum"], torch.from_numpy(z["weights_sum"])) and torch.equal(res["knife"], torch.from_numpy(z["knife"]))
    # the same seed draws the reference's vector (one torch.rand(N) at the first round)
    torch.manual_seed(m["seed"])
    seeded = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], **kw)
    assert torch.equal(seeded["noises"], noises) and torch.equal(seeded["rgb_map"], res["rgb_map"])


@pytest.mark.parametrize("dt_gamma", [0.0, 1.0 / 256])
def test_round_schedule_lemma_with_jittered_starts(oracle_ops, dt_gamma):
    from oracle import perturb
    from oracle.render import OracleModel
    for seed, ds, ms in ((0, 1.0, 8), (1, 32.0, 16), (2, 8.0, 16)):
        sc = scn.Scene(H=40, W=40, T=2, torso=False, max_steps=ms, density_scale=ds)
        hp = dict(sc.hparams, dt_gamma=dt_gamma)
        fi = sc.frame_inputs(1)
        ro, rd = fi["rays_o"].view(-1, 3), fi["rays_d"].view(-1, 3)
        N = ro.shape[0]
        noises = torch.rand(N, generator=torch.Generator().manual_seed(seed))
        orc = _oracle(sc, ds)
        ref = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], noises=noises,
                             bg_color=fi["bg_color"], T_thresh=0.01, **hp)
        B = ref["stats"]["B_total"]
        nears, fars = oracle_ops.near_far_from_aabb(ro, rd, sc.state["aabb_infer"], hp["min_near"])
        alive = torch.arange(N, dtype=torch.int32)
        rays_t = nears.clone()
        xyzs, dirs, deltas = perturb.march_rays(N, B, alive, rays_t, ro, rd, orc.bound, sc.state["density_bitfield"], orc.cascade,
                                                orc.grid_size, nears, fars, 128, True, dt_gamma, ms, noises=noises)
        sig, rgb, _ = orc.forward(xyzs, dirs, orc.cal_cond_feat(fi["cond"]), sc.state["individual_embeddings"][0])
        sig = sig * ds
        ws = torch.zeros(N); dp = torch.zeros(N); img = torch.zeros(N, 3)
        knife = torch.full((N,), float("inf")); n_samples = torch.zeros(N, dtype=torch.int32)
        ids = alive.long().clone()
        OracleModel._stats(ids, B, sig, deltas, ws.clone(), 0.01, knife, n_samples)
        oracle_ops.composite_rays(N, B, alive, rays_t, sig, rgb, deltas, ws, dp, img, 0.01)
        one = (img + (1 - ws).unsqueeze(-1) * fi["bg_color"].view(-1, 3)).clamp(0, 1)
        d = (one - ref["rgb_map"].view(-1, 3)).abs().max().item()
        assert d < 1e-6, (seed, dt_gamma, d)
        assert (ws - ref["weights_sum"]).abs().max().item() < 1e-6
        assert int(n_samples.sum()) == ref["stats"]["S"], (int(n_samples.sum()), ref["stats"]["S"])
        # the jitter is live: it moves samples (the unjittered single round differs)
        plain = orc.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], T_thresh=0.01, **hp)
        assert (plain["rgb_map"] - ref["rgb_map"]).abs().max().item() > 1e-4


def test_zero_noise_is_perturb_false(oracle_ops):
    from oracle import perturb
    for torso in (False, True):
        sc = scn.Scene(H=40, W=40, T=2, torso=torso, density_scale=8.0)
        fi = sc.frame_inputs(0)
        orc = _oracle(sc, 8.0)
        args = (fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"])
        a = perturb.render(orc, *args, noises=torch.zeros(sc.H * sc.W), bg_color=fi["bg_color"], T_thresh=0.01, **sc.hparams)
        b = orc.render(*args, bg_color=fi["bg_color"], T_thresh=0.01, **sc.hparams)
        for k in ("rgb_map", "depth_map", "weights_sum") + (("torso_rgb_map",) if torso else ()):
            assert torch.equal(a[k], b[k]), k
        assert a["stats"] == b["stats"]


def test_oracle_perturb_draws_once_per_render(oracle_ops):
    """One torch.rand(N) per render, at the first round; later rounds draw nothing (raymarching.py:388-392)."""
    from oracle import perturb
    sc = scn.Scene(H=32, W=32, T=2, torso=False, density_scale=16.0)
    fi = sc.frame_inputs(0)
    orc = _oracle(sc, 16.0)
    torch.manual_seed(5)
    res = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], T_thresh=0.01,
                         **sc.hparams)
    assert len(res["stats"]["schedule"]) > 1
    after = torch.rand(3)
    torch.manual_seed(5)
    first = torch.rand(32 * 32)
    assert torch.equal(res["noises"], first) and torch.equal(torch.rand(3), after)
