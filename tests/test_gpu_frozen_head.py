"""RADNeRF.frozen_head (gfpp.h section K) against the composed no-grad head block of the torso training step: near_far_from_aabb
(aabb_train) + march_rays_train + forward (train_precision "fp32") + composite_rays_train, with the same seed.

fp32 is held to 1e-5 max-abs, the bar golden (b) puts on the composed step; the tensor-core modes to the renderer's own bar
(1e-3 max-abs and 50 dB on the image, 1e-3 on weights_sum) against the fp32 composed path.  The scenes are
oracle/torso_train.golden_scene() (32 x 32) and a 256 x 256 torso scene."""
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200 import train_ops
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR
from oracle import torso_train as tt

pytestmark = pytest.mark.gpu

FP32_BAR = 1e-5
TC_BAR, TC_PSNR = 1e-3, 50.0
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_torso.npz")


def _model(sc, ds):
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale, m.mlp_precision = ds, "fp32"
    return m.cuda().train()


@pytest.fixture(scope="module")
def scenes():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import ops
    ops.build()
    out = {}
    for name, sc in (("golden", tt.golden_scene()), ("bench256", scn.Scene(H=256, W=256, T=4, torso=True, density_scale=tt.GOLDEN_DS))):
        m = _model(sc, tt.GOLDEN_DS)
        fi = sc.frame_inputs(tt.GOLDEN_FRAME)
        with torch.no_grad():
            feat = m.cal_cond_feat(fi["cond"].cuda())
        out[name] = {"sc": sc, "m": m, "ro": fi["rays_o"].cuda().reshape(-1, 3), "rd": fi["rays_d"].cuda().reshape(-1, 3), "feat": feat, "fi": fi}
    return out


def composed(m, ro, rd, feat, code, perturb=False, T_thresh=1e-4, max_steps=16, seed=0):
    """The no-grad block of oracle/torso_train.gfpp_train_step on the fp32 training ops (no step_counter)."""
    prec = m.mlp_precision
    m.mlp_precision = "fp32"
    try:
        torch.manual_seed(seed)
        with torch.no_grad():
            nears, fars = train_ops.near_far_from_aabb(ro, rd, m.aabb_train, m.min_near)
            counter = torch.zeros(2, dtype=torch.int32, device=ro.device)
            xyzs, dirs, deltas, rays = train_ops.march_rays_train(ro, rd, m.bound, m.density_bitfield, m.cascade, m.grid_size, nears, fars,
                                                                  counter, 0, perturb, 128, True, 0, max_steps)
            sig, rgb, amb = m(xyzs, dirs, feat, code)
            ws, _, _, img = train_ops.composite_rays_train(m.density_scale * sig, rgb, amb.abs().sum(-1), deltas, rays, T_thresh)
    finally:
        m.mlp_precision = prec
    return ws, img


def fused(m, ro, rd, feat, code, perturb=False, T_thresh=1e-4, max_steps=16, seed=0):
    torch.manual_seed(seed)
    return m.frozen_head(ro, rd, feat, code, perturb=perturb, T_thresh=T_thresh, max_steps=max_steps)


def _err(a, b):
    return (a - b).abs().max().item()


def _psnr(a, b):
    mse = ((a - b) ** 2).mean().item()
    return float("inf") if mse == 0 else 10 * np.log10(1.0 / mse)


@pytest.mark.parametrize("scene", ["golden", "bench256"])
@pytest.mark.parametrize("perturb", [False, True])
@pytest.mark.parametrize("T_thresh", [1e-4, 1e-2])
@pytest.mark.parametrize("max_steps", [4, 16])
@pytest.mark.parametrize("row", [0, 2])
def test_fp32_matches_composed(scenes, scene, perturb, T_thresh, max_steps, row):
    s = scenes[scene]
    m = s["m"]
    code = m.individual_embeddings[row]
    ws_c, img_c = composed(m, s["ro"], s["rd"], s["feat"], code, perturb, T_thresh, max_steps, seed=11)
    ws_f, img_f = fused(m, s["ro"], s["rd"], s["feat"], code, perturb, T_thresh, max_steps, seed=11)
    e_ws, e_img = _err(ws_f, ws_c), _err(img_f, img_c)
    hit = int((ws_c > 0).sum())
    print(f"\n[{scene} perturb={perturb} T_thresh={T_thresh} max_steps={max_steps} row={row}] {hit} rays hit; weights_sum {e_ws:.2e}, image {e_img:.2e}")
    assert hit > 0
    assert e_ws <= FP32_BAR and e_img <= FP32_BAR


def test_narrow_aabb_train_and_missing_rays(scenes):
    s = scenes["bench256"]
    m = s["m"]
    saved = m.aabb_train.clone()
    try:
        with torch.no_grad():
            m.aabb_train.copy_(m.aabb_infer * torch.tensor([0.6, 0.7, 0.6, 0.6, 0.7, 0.6], device="cuda"))
        code = m.individual_embeddings[2]
        ws_c, img_c = composed(m, s["ro"], s["rd"], s["feat"], code)
        ws_f, img_f = fused(m, s["ro"], s["rd"], s["feat"], code)
        print(f"\n[aabb_train narrower than aabb_infer] weights_sum {_err(ws_f, ws_c):.2e}, image {_err(img_f, img_c):.2e}")
        assert _err(ws_f, ws_c) <= FP32_BAR and _err(img_f, img_c) <= FP32_BAR
    finally:
        with torch.no_grad():
            m.aabb_train.copy_(saved)
    # the narrow box cuts samples that the full one keeps
    ws_full, _ = fused(m, s["ro"], s["rd"], s["feat"], m.individual_embeddings[2])
    assert not torch.equal(ws_full, ws_f)
    # rays that miss the volume: exact zeros
    N = s["ro"].shape[0]
    ro = torch.tensor([[0.0, 0.0, 5.0]], device="cuda").expand(N, 3).contiguous()
    rd = torch.nn.functional.normalize(torch.rand(N, 3, device="cuda") + 0.1, dim=-1)   # pointing away from the volume
    ws, img = fused(m, ro, rd, s["feat"], m.individual_embeddings[2])
    assert torch.count_nonzero(ws) == 0 and torch.count_nonzero(img) == 0


@pytest.mark.parametrize("scene", ["golden", "bench256"])
@pytest.mark.parametrize("precision", ["fp16", "robust", "bf16x3", "bf16"])
def test_tensor_core_modes_against_fp32_composed(scenes, scene, precision):
    s = scenes[scene]
    m = s["m"]
    code = m.individual_embeddings[2]
    ws_c, img_c = composed(m, s["ro"], s["rd"], s["feat"], code, perturb=True, seed=5)
    m.mlp_precision = precision
    try:
        ws_f, img_f = fused(m, s["ro"], s["rd"], s["feat"], code, perturb=True, seed=5)
    finally:
        m.mlp_precision = "fp32"
    e_ws, e_img, p = _err(ws_f, ws_c), _err(img_f, img_c), _psnr(img_f, img_c)
    print(f"\n[{scene} {precision}] weights_sum {e_ws:.2e}, image {e_img:.2e}, PSNR {p:.1f} dB")
    assert e_ws <= TC_BAR and e_img <= TC_BAR and p > TC_PSNR


def test_determinism_sync_free_no_grad_and_render_untouched(scenes):
    s = scenes["bench256"]
    m = s["m"]
    code = m.individual_embeddings[2]
    a = fused(m, s["ro"], s["rd"], s["feat"], code, perturb=True, seed=3)
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = fused(m, s["ro"], s["rd"], s["feat"], code, perturb=True, seed=3)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not a[0].requires_grad and not a[1].requires_grad and code.requires_grad
    # render() in eval mode is not affected by a frozen_head call with another code row
    fi = s["fi"]
    kw = dict(rays_o=fi["rays_o"].cuda(), rays_d=fi["rays_d"].cuda(), cond=fi["cond"].cuda(), bg_coords=fi["bg_coords"].cuda(),
              poses=fi["poses"].cuda(), bg_color=fi["bg_color"].cuda())
    m.eval()
    try:
        r0 = m.render(**kw)
        fused(m, s["ro"], s["rd"], s["feat"], code)
        r1 = m.render(**kw)
    finally:
        m.train()
    for k in ("rgb_map", "weights_sum", "depth_map"):
        assert torch.equal(r0[k], r1[k]), k
    # the step counters are left alone
    assert m.local_step == 0 and int(m.step_counter.abs().sum()) == 0


def _frozen_step(model, rays_o, rays_d, cond, bg_coords, poses, index, bg_color, max_steps):
    """oracle/torso_train.gfpp_train_step with its no-grad head block replaced by frozen_head."""
    rays_o, rays_d, bg_coords = rays_o.reshape(-1, 3), rays_d.reshape(-1, 3), bg_coords.reshape(-1, 2)
    with torch.no_grad():
        cond_feat = model.cal_cond_feat(cond)
    weights_sum, image = model.frozen_head(rays_o, rays_d, cond_feat, model.individual_embeddings[index], max_steps=max_steps)
    mask = model.torso_mask(bg_coords)
    N = rays_o.shape[0]
    torso_alpha = torch.zeros(N, 1, device=rays_o.device)
    torso_color = torch.zeros(N, 3, device=rays_o.device)
    alpha, color, deform = model.forward_torso(bg_coords[mask], poses, model.torso_individual_codes[index])
    torso_alpha[mask] = alpha
    torso_color[mask] = color
    bg = torso_color * torso_alpha + bg_color.reshape(-1, 3) * (1 - torso_alpha)
    rgb = (image + (1 - weights_sum).unsqueeze(-1) * bg).clamp(0, 1)
    return {"torso_alpha_map": torso_alpha, "torso_rgb_map": bg, "rgb_map": rgb, "weights_sum": weights_sum, "deform": deform}


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def test_torso_step_with_frozen_head_against_golden_b(scenes):
    """The torso training step on frozen_head meets golden (b): its maps within 1e-5 and its torso gradients as close to the float64
    gradients as the composed step's (test_gpu_torso_train.py's bar: twice the reference's own fp32 error, floor 1e-5)."""
    m = scenes["golden"]["m"]
    z = np.load(GOLDEN)
    inp = {k: torch.from_numpy(z[f"b.{k}"]).cuda() for k in ("rays_o", "rays_d", "cond", "bg_coords", "bg_color", "gt")}
    index = torch.tensor([tt.GOLDEN_INDEX], device="cuda")
    pose6 = torch.from_numpy(z["pose6"]).cuda()
    m.zero_grad(set_to_none=True)
    res = _frozen_step(m, inp["rays_o"], inp["rays_d"], inp["cond"], inp["bg_coords"], pose6, index, inp["bg_color"], tt.GOLDEN_MAX_STEPS)
    tt.task_loss(res, inp["gt"], tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    torch.cuda.synchronize()
    for k in ("torso_alpha_map", "torso_rgb_map", "rgb_map", "weights_sum"):
        e = _rel(res[k].detach().reshape(-1), z[f"b.{k}"].reshape(-1))
        print(f"golden (b) with frozen_head {k}: rel {e:.2e}")
        assert e <= 1e-5, (k, e)
    params = dict(m.named_parameters())
    assert all(p.grad is None for k, p in params.items() if k not in tt.TRAINABLE + ["torso_individual_codes"]), "the head must stay frozen"
    grads = {k: params[k].grad for k in tt.TRAINABLE[:6]}
    grads["code"] = params["torso_individual_codes"].grad[tt.GOLDEN_INDEX]
    for k, g in grads.items():
        e = _rel(g, z[f"b.grad64.{k}"])
        e_ref = _rel(z[f"b.grad.{k}"], z[f"b.grad64.{k}"])
        print(f"golden (b) with frozen_head {k}: to float64 {e:.2e}, reference {e_ref:.2e}")
        assert e <= max(2 * e_ref, 1e-5), (k, e, e_ref)
    m.zero_grad(set_to_none=True)


def test_torso_sr_model_matches_its_composed_head():
    """A RADNeRFTorsowithSR model (the torso-SR golden's hparams: eye-blink conditioning) at the fp32 bar, with the eye area in
    cond_feat."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import torso_sr_train as tst
    hp = tst.golden_hparams("b")
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(tst.golden_state(hp), strict=False)
    m.density_scale, m.mlp_precision = tt.GOLDEN_DS, "fp32"
    m = m.cuda().train()
    sc = scn.Scene(H=64, W=64, T=4, torso=True)
    with torch.no_grad():
        m.density_bitfield.copy_(sc.state["density_bitfield"].cuda())
    fi = sc.frame_inputs(1)
    ro, rd = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
    with torch.no_grad():
        feat = m.cal_cond_feat(scn.cond_window(sc.cond, 1, hp["smo_win_size"]).cuda(), eye_area_percent=torch.tensor([0.3], device="cuda"))
    code = m.individual_embeddings[1]
    ws_c, img_c = composed(m, ro, rd, feat, code)
    ws_f, img_f = fused(m, ro, rd, feat, code)
    print(f"\n[torso-SR] {int((ws_c > 0).sum())} rays hit; weights_sum {_err(ws_f, ws_c):.2e}, image {_err(img_f, img_c):.2e}")
    assert int((ws_c > 0).sum()) > 0
    assert _err(ws_f, ws_c) <= FP32_BAR and _err(img_f, img_c) <= FP32_BAR
