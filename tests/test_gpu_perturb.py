"""perturb=True in the inference renderer on the GPU: jittered ray starts in k_ray_setup (gfpp_frames.noises).

Bars as tests/test_gpu_render.py: rgb / alpha within 1e-3 max-abs (knife-edge rays reported and excluded), PSNR >= 50 dB; the
discrete by-products B (round-schedule cap), S (evaluated samples) and P (torso pixels) exactly equal."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from helpers import build_model, parity_report

pytestmark = pytest.mark.gpu

TOL = 1e-3
PSNR_MIN = 50.0
GOLD = os.path.join(os.path.dirname(__file__), "golden")
GOLDEN = sorted(glob.glob(os.path.join(GOLD, "perturb_*.npz")))
PRECISIONS = ["fp32", "fp16", "robust", "bf16x3", "bf16"]


def _cuda(fi):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in fi.items()}


def _frames(model, fi, hp, T_thresh, torso, noise=None, **extra):
    cf = model.cal_cond_feat(fi["cond"]).view(1, -1)
    return model.render_frames(cf, rays_o=fi["rays_o"], rays_d=fi["rays_d"], pose6=fi["poses"] if torso else None,
                               bg_coords=fi["bg_coords"] if torso else None, bg_color=fi["bg_color"], dt_gamma=hp["dt_gamma"],
                               max_steps=hp["max_steps"], T_thresh=T_thresh, noise=noise, **extra)


def _check(out, ref, knife, torso, label):
    rep = parity_report(out["rgb_map"].reshape(-1, 3), ref["rgb_map"].reshape(-1, 3), knife)
    print(f"[{label}] rgb max|d|={rep['max_abs']:.2e} (all {rep['max_abs_all']:.2e}, knife-edge rays {rep['n_knife']}, >1e-3: {rep['n_over']}) "
          f"psnr={rep['psnr']:.1f} dB")
    assert rep["max_abs"] <= TOL and rep["psnr"] >= PSNR_MIN, (label, rep)
    assert rep["n_over"] <= max(2, rep["n_knife"]), "errors above tolerance must be explained by knife-edge rays"
    if "weights_sum" in ref:
        repw = parity_report(out["weights_sum"].reshape(-1), ref["weights_sum"].reshape(-1), knife)
        assert repw["max_abs"] <= TOL, (label, repw)
    d_ref, d_out = ref["depth_map"].reshape(-1).float().cpu(), out["depth_map"].reshape(-1).cpu()
    assert torch.equal(torch.isnan(d_ref), torch.isnan(d_out))
    ok = ~torch.isnan(d_ref) & (knife.reshape(-1) >= 1e-3)
    assert (d_ref[ok] - d_out[ok]).abs().max().item() <= 2e-3
    if torso:
        for k in ("torso_alpha_map", "torso_rgb_map"):
            d = (out[k].cpu().reshape(-1) - ref[k].reshape(-1).cpu()).abs().max().item()
            assert d <= TOL, (label, k, d)


# ------------------------------------------------------------------------------------------------ 1. the reference's own goldens
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_matches_reference_golden(path):
    z = np.load(path)
    m = json.loads(bytes(z["meta"]).decode())
    torso = m["torso"]
    sc = scn.Scene(H=m["size"], W=m["size"], T=8, torso=torso, max_steps=m["max_steps"], density_scale=m["density_scale"])
    hp = sc.hparams
    model = build_model(sc)
    fi = _cuda(sc.frame_inputs(m["frame"]))
    noise = torch.from_numpy(z["noises"]).cuda()
    ref = {k: torch.from_numpy(z[k]) for k in z.files if k not in ("meta", "noises", "knife")}
    knife = torch.from_numpy(z["knife"])
    res = _frames(model, fi, hp, m["T_thresh"], torso, noise=noise, want_stats=True)
    st = res["stats"][0].tolist()
    print(f"[{m['name']}] B={st[0]} survivors={st[1]} S={st[2]} P={st[3]} (reference B={m['stats']['B_total']} S={m['stats']['S']} P={m['stats']['P']})")
    assert (st[0], st[2], st[3]) == (m["stats"]["B_total"], m["stats"]["S"], m["stats"]["P"])
    _check(res, ref, knife, torso, f"{m['name']} render_frames fp32")
    # the render() API with the golden's draw in place of the device draw (the draw itself is pinned by test_rng_semantics)
    model._ray_start_noise = lambda n: noise.clone()
    out = model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=m["frame"], staged=False,
                       bg_color=fi["bg_color"], perturb=True, force_all_rays=False, T_thresh=m["T_thresh"], **hp)
    _check(out, ref, knife, torso, f"{m['name']} render() fp32")
    assert torch.equal(out["rgb_map"].view(-1, 3), res["rgb_map"].view(-1, 3))


# ------------------------------------------------------------------------------------------------ 2. every mode vs the oracle
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("torso,ds", [(False, 16.0), (True, 8.0)], ids=["head", "torso"])
def test_every_mode_matches_oracle_with_shared_noise(oracle_ops, precision, torso, ds):
    from oracle import perturb
    from oracle.render import OracleModel
    sc = scn.Scene(H=64, W=64, T=4, torso=torso, density_scale=ds)
    fi = sc.frame_inputs(1)
    noise = torch.rand(64 * 64, generator=torch.Generator().manual_seed(7))
    orc = OracleModel(sc.state, sc.hparams)
    orc.density_scale = ds
    ref = perturb.render(orc, fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], noises=noise, bg_color=fi["bg_color"],
                         T_thresh=sc.T_thresh, **sc.hparams)
    model = build_model(sc, precision=precision)
    res = _frames(model, _cuda(fi), sc.hparams, sc.T_thresh, torso, noise=noise.cuda(), want_stats=True)
    _check(res, ref, ref["knife"], torso, f"{precision} torso={torso} ds={ds}")
    st = res["stats"][0].tolist()
    n_knife = int((ref["knife"] < 1e-3).sum())
    assert abs(st[2] - ref["stats"]["S"]) <= n_knife and st[3] == ref["stats"]["P"], (st, ref["stats"])


# ------------------------------------------------------------------------------------------------ 3. zero noise, argument checks
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("torso", [False, True])
def test_zero_noise_is_bit_identical_to_no_perturb(precision, torso):
    sc = scn.Scene(H=64, W=64, T=4, torso=torso, density_scale=8.0)
    model = build_model(sc, precision=precision)
    fi = _cuda(sc.frame_inputs(2))
    a = _frames(model, fi, sc.hparams, sc.T_thresh, torso, want_stats=True)
    b = _frames(model, fi, sc.hparams, sc.T_thresh, torso, noise=torch.zeros(64 * 64, device="cuda"), want_stats=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    with pytest.raises(ValueError, match="noise"):
        _frames(model, fi, sc.hparams, sc.T_thresh, torso, noise=torch.zeros(64 * 64 - 1, device="cuda"))
    with pytest.raises(ValueError, match="noise"):
        _frames(model, fi, sc.hparams, sc.T_thresh, torso, noise=torch.zeros(2, 64 * 64, device="cuda"))


# ------------------------------------------------------------------------------------------------ 4./5. RNG semantics, determinism
@pytest.mark.parametrize("torso", [False, True])
def test_rng_semantics_and_run_to_run(torso):
    sc = scn.Scene(H=64, W=64, T=4, torso=torso, density_scale=8.0)
    model = build_model(sc)
    fi = _cuda(sc.frame_inputs(1))
    N = 64 * 64

    def render(seed):
        torch.cuda.manual_seed(seed)
        out = model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], perturb=True,
                           T_thresh=sc.T_thresh, **sc.hparams)
        return out, torch.cuda.get_rng_state()

    out, state = render(3)
    torch.cuda.manual_seed(3)
    noise = torch.rand(N, device="cuda")
    assert torch.equal(state, torch.cuda.get_rng_state()), "render(perturb=True) must consume exactly one N-draw"
    res = _frames(model, fi, sc.hparams, sc.T_thresh, torso, noise=noise)
    for k in ("rgb_map", "depth_map", "weights_sum") + (("torso_alpha_map",) if torso else ()):
        assert torch.equal(out[k].reshape(-1), res[k].reshape(-1)), k
    again, _ = render(3)
    for k in out:
        assert torch.equal(out[k], again[k]), k
    other, _ = render(4)
    assert not torch.equal(other["rgb_map"], out["rgb_map"])
    # perturb=False draws nothing
    torch.cuda.manual_seed(3)
    model.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], perturb=False,
                 T_thresh=sc.T_thresh, **sc.hparams)
    after = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(3)
    assert torch.equal(after, torch.cuda.get_rng_state())


def _head_sr():
    from genefaceplusplus_b200.renderer import RADNeRFwithSR
    z = np.load(os.path.join(GOLD, "head_sr256.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    hp = may_hparams(**meta["overrides"])
    m = RADNeRFwithSR(hp)
    m.load_state_dict(scn.make_head_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    return m.cuda().eval(), hp, meta


def _torso_sr():
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
    z = np.load(os.path.join(GOLD, "torso_sr256.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    hp = may_hparams(**{**meta["overrides"], "torso_head_aware": True})
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    return m.cuda().eval(), hp, meta


def _validation_call(m, hp, torso, t=3, **extra):
    """The reference's validation_step (tasks/radnerfs/radnerf*.py run_model(sample, infer=False) in eval mode under no_grad)."""
    R = 256
    sc = scn.Scene(H=R, W=R, T=8, torso=torso, density_scale=m.density_scale)
    fi = _cuda(sc.frame_inputs(t))
    cond = scn.cond_window(sc.cond, t, hp["smo_win_size"]).cuda()
    kw = dict(hp)
    kw["max_steps"] = 16
    with torch.no_grad():
        return m.render(fi["rays_o"], fi["rays_d"], cond, fi["bg_coords"], fi["poses"], index=t, staged=False, bg_color=fi["bg_color"],
                        perturb=True, force_all_rays=False, cond_mask=None, **{**kw, **extra}), fi, cond


@pytest.mark.parametrize("which", ["head_sr", "torso_sr"])
def test_sr_classes_draw_the_marching_noise_before_the_sr_noise(which):
    """The reference marches first (its step-0 draw) and runs the SR head's noise_mode="random" planes afterwards: record the
    generator state at the marching draw and at every SR call, then replay both by hand."""
    torso = which == "torso_sr"
    m, hp, meta = _torso_sr() if torso else _head_sr()
    N = 256 * 256
    log = []
    draw = m._ray_start_noise
    m._ray_start_noise = lambda n: (log.append(("march", torch.cuda.get_rng_state())), draw(n))[1]
    sr_forward = m.sr_net.forward

    def sr_logged(x, *a, **k):
        log.append(("sr", torch.cuda.get_rng_state(), x.detach().clone()))
        return sr_forward(x, *a, **k)

    m.sr_net.forward = sr_logged
    extra = {"lm68": scn.lm68_sequence(8)[3].reshape(1, 136).cuda(), "upscale_torso": True} if torso else {}
    torch.cuda.manual_seed(21)
    out, fi, cond = _validation_call(m, hp, torso, eye_area_percent=torch.tensor([[meta["eye"]]]), **extra)
    end = torch.cuda.get_rng_state()
    assert [e[0] for e in log] == ["march", "sr"] + (["sr"] if torso else [])
    torch.cuda.manual_seed(21)
    assert torch.equal(log[0][1], torch.cuda.get_rng_state())
    noise = torch.rand(N, device="cuda")
    assert torch.equal(log[1][1], torch.cuda.get_rng_state()), "the SR head must draw after the marching noise"
    # replay: the head image from the same noise vector, then the SR head from the state right after the N-draw
    cf = m.cal_cond_feat(cond, eye_area_percent=torch.tensor([[meta["eye"]]]))
    zero = torch.zeros(N, 3, device="cuda") if torso else fi["bg_color"]
    hd = m.render_frames(cf.view(1, -1), rays_o=fi["rays_o"], rays_d=fi["rays_d"], bg_color=zero, dt_gamma=hp["dt_gamma"], max_steps=16,
                         T_thresh=1e-4, noise=noise)
    assert torch.equal(hd["depth_map"].view(-1), out["depth_map"].view(-1))
    if not torso:
        assert torch.equal(hd["rgb_map"].view(1, 256, 256, 3).permute(0, 3, 1, 2), out["rgb_map"])
    m.sr_net.forward = sr_forward
    with torch.no_grad():
        for entry, key in zip(log[1:], ("sr_rgb_map", "sr_torso_rgb_map")):
            torch.cuda.set_rng_state(entry[1])
            sr = m.sr_net(entry[2], noise_mode="random").clamp(0, 1)
            d = (sr - out[key]).abs().max().item()
            print(f"[{which}] replayed {key}: max|d| = {d:.2e}")
            assert d <= 1e-5, (key, d)
    # and the render consumed nothing after the SR head's planes
    assert torch.equal(torch.cuda.get_rng_state(), end)


# ------------------------------------------------------------------------------------------------ 6. multi-frame noise [F,N]
@pytest.mark.parametrize("torso", [False, True])
def test_multi_frame_noise_equals_single_frame_calls(torso):
    sc = scn.Scene(H=48, W=48, T=4, torso=torso, density_scale=8.0)
    model = build_model(sc)
    N, F = 48 * 48, 3
    fis = [_cuda(sc.frame_inputs(t)) for t in range(F)]
    noise = torch.rand(F, N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    cf = torch.cat([model.cal_cond_feat(fi["cond"]).view(1, -1) for fi in fis])
    cat = lambda k: torch.cat([fi[k].reshape(1, -1, fi[k].shape[-1]) for fi in fis])
    multi = model.render_frames(cf, rays_o=cat("rays_o"), rays_d=cat("rays_d"), pose6=cat("poses").view(F, 6) if torso else None,
                                bg_coords=fis[0]["bg_coords"] if torso else None, bg_color=fis[0]["bg_color"], dt_gamma=sc.hparams["dt_gamma"],
                                max_steps=sc.hparams["max_steps"], T_thresh=sc.T_thresh, noise=noise, want_stats=True)
    survivors = 0
    for f in range(F):
        one = _frames(model, fis[f], sc.hparams, sc.T_thresh, torso, noise=noise[f], want_stats=True)
        for k in one:
            if k == "stats":    # (B, survivors, S, P): the survivor count is the call's total over its frames
                assert torch.equal(multi[k][f, [0, 2, 3]], one[k][0, [0, 2, 3]]), (f, multi[k][f], one[k][0])
                survivors += int(one[k][0, 1])
            else:
                assert torch.equal(multi[k][f], one[k][0]), (f, k)
    assert int(multi["stats"][0, 1]) == survivors


# ------------------------------------------------------------------------------------------------ 7. the reference's validation call
def test_validation_step_call_for_all_four_classes():
    from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso
    N = 256 * 256
    for torso in (False, True):
        sc = scn.Scene(H=64, W=64, T=8, torso=torso, density_scale=8.0)
        m = build_model(sc)
        assert isinstance(m, RADNeRFTorso if torso else RADNeRF)
        fi = _cuda(sc.frame_inputs(2))
        with torch.no_grad():
            out = m.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], index=2, staged=False, bg_color=fi["bg_color"],
                           perturb=True, force_all_rays=False, cond_mask=None, **sc.hparams)
        n = 64 * 64
        assert out["rgb_map"].shape == fi["rays_o"].shape and out["depth_map"].shape == fi["rays_o"].shape[:-1]
        if torso:
            assert out["torso_alpha_map"].shape == (n, 1) and out["torso_rgb_map"].shape[-1] == 3 and out["deform"].shape[-1] == 2
        assert torch.isfinite(out["rgb_map"]).all()
    m, hp, meta = _head_sr()
    out, _, _ = _validation_call(m, hp, False, eye_area_percent=torch.tensor([[meta["eye"]]]))
    assert out["rgb_map"].shape == (1, 3, 256, 256) and out["sr_rgb_map"].shape == (1, 3, 512, 512)
    assert out["depth_map"].shape == (1, N)
    m, hp, meta = _torso_sr()
    out, _, _ = _validation_call(m, hp, True, eye_area_percent=torch.tensor([[meta["eye"]]]),
                                 lm68=scn.lm68_sequence(8)[3].reshape(1, 136).cuda(), upscale_torso=True)
    assert out["rgb_map"].shape == (1, 3, 256, 256) and out["sr_rgb_map"].shape == (1, 3, 512, 512)
    assert out["torso_rgb_map"].shape == (1, 3, 256, 256) and out["sr_torso_rgb_map"].shape == (1, 3, 512, 512)
    assert out["torso_alpha_map"].shape == (N, 1) and out["depth_map"].shape == (1, N)
    for k in ("rgb_map", "sr_rgb_map", "sr_torso_rgb_map"):
        assert torch.isfinite(out[k]).all() and out[k].min().item() >= 0 and out[k].max().item() <= 1
