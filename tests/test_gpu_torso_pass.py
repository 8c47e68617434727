"""torso_pass() of both torso models (gfpp.h section M around the training fields of sections H and I) against the composed recipe of
the torso training steps (oracle/torso_train.gfpp_train_step's torso block and its torso-SR counterpart in README):
  1. the mask and compaction exactly (slot, idx, gathers) on the golden scene, full bg_coords grids, random coords with points outside
     [-1,1] and on grid nodes, thresholds with ties, below and above every occupancy;
  2. the maps and deform bit-identical, every background kind, both SR parts (head-aware with a code; neither);
  3. golden (b) of tests/golden/train_torso.npz with frozen_head;
  4. gradients within 1e-5 of max|grad| of the composed recipe's, for both task losses and the SR deform term, with pixels whose
     pre-clamp rgb_map is exactly 0 or 1;
  5. three Adam steps at 65 536 rays with the fp16 frozen head under autocast and a GradScaler;
  6. determinism, and M == 0.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.renderer import RADNeRFTorso, RADNeRFTorsowithSR
from oracle import torso_sr_train as tst
from oracle import torso_train as tt

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_torso.npz")
STEP_OUT = 1e-5          # golden (b): maps
FLOOR = 1e-5             # golden (b): gradient bar's floor, relative to max|float64 gradient|
GRAD_REL = 1e-5          # gradients against the composed recipe, relative to its max|grad|
ADAM_LOSS_REL = 1e-3     # three Adam steps: loss (the bar of test_gpu_torso_train.py's Adam test)
ADAM_PARAM_REL = 5e-2    # three Adam steps: parameters, relative L2
LAMBDA_DEFORM = 1e-3     # lambda_torso_deform of the torso-SR configs


def _torso(sc, ds=tt.GOLDEN_DS):
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    m.density_scale, m.mlp_precision = ds, "fp32"
    return m.cuda().train()


def _sr(part, scene=None):
    hp = tst.golden_hparams(part)
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(tst.golden_state(hp), strict=False)
    m.density_scale, m.mlp_precision = tt.GOLDEN_DS, "fp32"
    m = m.cuda().train()
    if scene is not None:
        with torch.no_grad():
            m.density_bitfield.copy_(scene.state["density_bitfield"].cuda())
    return m


@pytest.fixture(scope="module")
def golden():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from oracle import ops
    ops.build()
    sc = tt.golden_scene()
    m = _torso(sc)
    fi = sc.frame_inputs(tt.GOLDEN_FRAME)
    with torch.no_grad():
        feat = m.cal_cond_feat(fi["cond"].cuda())
    ro, rd = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
    ws, img = m.frozen_head(ro, rd, feat, m.individual_embeddings[tt.GOLDEN_INDEX], max_steps=tt.GOLDEN_MAX_STEPS)
    return {"sc": sc, "m": m, "fi": fi, "ws": ws, "img": img, "bg_coords": fi["bg_coords"].cuda().reshape(-1, 2),
            "pose6": fi["poses"].cuda(), "index": torch.tensor([tt.GOLDEN_INDEX], device="cuda")}


# ------------------------------------------------------------------------------------------------ the composed recipes
def _composite(mask, alpha, color, image, ws, bg_color):
    N = mask.shape[0]
    ta = torch.zeros(N, 1, device="cuda")
    tc = torch.zeros(N, 3, device="cuda")
    ta[mask] = alpha
    tc[mask] = color
    bg = 1 if bg_color is None else bg_color.reshape(-1, 3)
    trgb = tc * ta + bg * (1 - ta)
    rgb = (image + (1 - ws).unsqueeze(-1) * trgb).clamp(0, 1)
    return {"torso_alpha_map": ta, "torso_rgb_map": trgb, "rgb_map": rgb, "weights_sum": ws}


def composed_torso(m, image, ws, bg_coords, pose6, code, bg_color):
    """The torso block of oracle/torso_train.gfpp_train_step."""
    mask = m.torso_mask(bg_coords)
    alpha, color, deform = m.forward_torso(bg_coords[mask], pose6, code)
    res = _composite(mask, alpha, color, image, ws, bg_color)
    if bool(mask.any()):
        res["deform"] = deform
    return res


def composed_sr(m, image, ws, bg_coords, code, bg_color, lm68):
    """README's torso-SR step (radnerf_torso_sr.py:196-221) with the same composite."""
    G = m.grid_size
    occ = F.grid_sample(m.density_grid_torso.view(1, 1, G, G), bg_coords.view(1, -1, 1, 2), align_corners=True).view(-1)
    mask = occ > min(m.density_thresh_torso, m.mean_density_torso)
    alpha, color, deform = m.forward_torso(bg_coords[mask], None, code, image[mask], ws[mask].unsqueeze(-1), lm68=lm68)
    res = _composite(mask, alpha, color, image, ws, bg_color)
    res["deform"] = deform
    return res


def _native_mask(m, bg_coords, image=None, ws=None):
    L = _capi.lib()
    xy = bg_coords.reshape(-1, 2).float().contiguous()
    N = xy.shape[0]
    i32 = torch.int32
    idx, slot, count = torch.empty(N, dtype=i32, device="cuda"), torch.empty(N, dtype=i32, device="cuda"), torch.empty(1, dtype=i32, device="cuda")
    xy_m = torch.empty(N, 2, device="cuda")
    img_m = torch.empty(N, 3, device="cuda") if image is not None else None
    ws_m = torch.empty(N, device="cuda") if image is not None else None
    work = torch.empty(L.gfpp_torso_pass_workspace_bytes(N), dtype=torch.uint8, device="cuda")
    thr = float(min(m.density_thresh_torso, m.mean_density_torso))
    p = (lambda t: None if t is None else t.data_ptr())
    _capi.check(L.gfpp_torso_mask(m.density_grid_torso.data_ptr(), m.grid_size, thr, xy.data_ptr(), N, p(image), p(ws), idx.data_ptr(),
                                  slot.data_ptr(), xy_m.data_ptr(), p(img_m), p(ws_m), count.data_ptr(), work.data_ptr(), work.numel(),
                                  _capi.stream_ptr()), "gfpp_torso_mask")
    M = int(count.item())
    return slot, idx[:M], xy_m[:M], None if img_m is None else img_m[:M], None if ws_m is None else ws_m[:M]


# ------------------------------------------------------------------------------------------------ 1. mask
def _coords_sets(G):
    g = torch.Generator().manual_seed(17)
    nodes = (-1 + 2 * torch.arange(G, dtype=torch.float32) / (G - 1))
    ny, nx = torch.meshgrid(nodes, nodes, indexing="ij")
    rnd = torch.rand(200000, 2, generator=g) * 2.4 - 1.2                  # a sixth of them outside [-1,1]
    edges = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [-1.0, 1.0], [0.0, 0.0], [1.0, 0.5], [-1.0000001, 0.2], [1.0000001, -0.3]])
    return {"golden32": None, "grid256": scn.get_bg_coords(256, 256), "grid512": scn.get_bg_coords(512, 512),
            "random+nodes": torch.cat([rnd, torch.stack([nx, ny], -1).reshape(-1, 2), edges])}


@pytest.mark.parametrize("grid", ["binary", "levels"])
@pytest.mark.parametrize("thr", ["default", "tie", "below_all", "above_all"])
def test_mask_and_compaction_match_torso_mask(golden, grid, thr):
    m = golden["m"]
    saved = (m.density_grid_torso.clone(), m.density_thresh_torso, m.mean_density_torso)
    try:
        G = m.grid_size
        if grid == "levels":     # values in {0, .25, .5, .75, 1}: interpolated occupancies hit them exactly at nodes and in flat cells
            q = torch.randint(0, 5, (G // 8, G // 8), generator=torch.Generator().manual_seed(3)).float() / 4
            m.density_grid_torso.copy_(q.repeat_interleave(8, 0).repeat_interleave(8, 1).reshape(-1).cuda())
        vals = {"default": (0.01, 0.0), "tie": (10.0, 0.5 if grid == "levels" else 1.0), "below_all": (10.0, -1.0), "above_all": (10.0, 2.0)}
        m.density_thresh_torso, m.mean_density_torso = vals[thr]
        for name, coords in _coords_sets(G).items():
            xy = golden["bg_coords"] if coords is None else coords.cuda().reshape(-1, 2)
            mask = m.torso_mask(xy)
            img = torch.rand(xy.shape[0], 3, device="cuda")
            wsum = torch.rand(xy.shape[0], device="cuda")
            slot, idx, xy_m, img_m, ws_m = _native_mask(m, xy, img, wsum)
            M = idx.shape[0]
            print(f"[{grid} {thr} {name}] N={xy.shape[0]} M={M}")
            bad = (slot >= 0) != mask
            if grid == "levels" and thr == "tie":
                # F.grid_sample(align_corners=True) runs on cuDNN's sampler, whose rounding is not public: on a multi-level grid an
                # occupancy that ties the threshold may come out one ulp apart.  Disagreements are allowed there and only there.
                t = torch.tensor(vals[thr][1], device="cuda")
                occ = F.grid_sample(m.density_grid_torso.view(1, 1, G, G), xy.view(1, -1, 1, 2), align_corners=True).view(-1)
                near = (occ == t) | (occ == torch.nextafter(t, t + 1)) | (occ == torch.nextafter(t, t - 1))
                print(f"  {int(bad.sum())} disagreement(s) among {int(near.sum())} pixels within one ulp of the threshold")
                assert not bool((bad & ~near).any()), name
                mask = slot >= 0                       # the compaction is checked against the kernel's own mask
            assert int(((slot >= 0) != mask).sum()) == 0, (name, int(bad.sum()))
            assert torch.equal(idx.long(), mask.nonzero().reshape(-1)), name
            assert torch.equal(slot[idx.long()], torch.arange(M, dtype=torch.int32, device="cuda"))
            assert torch.equal(xy_m, xy[mask]) and torch.equal(img_m, img[mask]) and torch.equal(ws_m, wsum[mask])
            if thr == "below_all":
                assert M == xy.shape[0]
            if thr == "above_all":
                assert M == 0
    finally:
        m.density_grid_torso.copy_(saved[0])
        m.density_thresh_torso, m.mean_density_torso = saved[1], saved[2]


# ------------------------------------------------------------------------------------------------ 2. forward, bit-identical
def _bg(kind, N):
    if kind == "none":
        return None
    if kind == "colour":
        return torch.tensor([0.2, 0.5, 0.9], device="cuda")
    return torch.rand(1, N, 3, generator=torch.Generator(device="cuda").manual_seed(8), device="cuda")


def _assert_equal_maps(res, ref, keys=("torso_alpha_map", "torso_rgb_map", "rgb_map", "deform")):
    for k in keys:
        assert res[k].shape == ref[k].shape, k
        assert torch.equal(res[k].detach(), ref[k].detach()), (k, (res[k] - ref[k]).abs().max().item())


@pytest.mark.parametrize("bg", ["none", "colour", "per_pixel"])
def test_torso_forward_bit_identical(golden, bg):
    s = golden
    m = s["m"]
    N = s["bg_coords"].shape[0]
    code = m.torso_individual_codes[s["index"]]
    bgc = _bg(bg, N)
    res = m.torso_pass(s["img"], s["ws"], s["bg_coords"], s["pose6"], code, bg_color=bgc)
    assert m.last_launch_count == 3 + 2 + 1          # mask, field forward (relayout + query), composite
    ref = composed_torso(m, s["img"], s["ws"], s["bg_coords"], s["pose6"], code, bgc)
    print(f"\n[{bg}] M = {ref['deform'].shape[0]} of {N}")
    _assert_equal_maps(res, ref)
    assert res["torso_alpha_map"].requires_grad and res["deform"].requires_grad


def _sr_inputs(part, N_side=64):
    m = _sr(part)
    N = N_side * N_side
    g = torch.Generator(device="cuda").manual_seed(21)
    ws = torch.rand(N, generator=g, device="cuda")
    img = torch.rand(N, 3, generator=g, device="cuda") * ws[:, None]
    bgc = scn.get_bg_coords(N_side, N_side).cuda().reshape(-1, 2)
    row = torch.tensor([tst.GOLDEN_INDEX], device="cuda")
    code = (lambda: m.torso_individual_codes[row] if m.torso_individual_embedding_dim else None)   # a fresh index node per graph
    return m, img, ws, bgc, code, tst.golden_lm68().cuda()


@pytest.mark.parametrize("part", ["b", "c"])
@pytest.mark.parametrize("bg", ["none", "colour", "per_pixel"])
def test_sr_forward_bit_identical(part, bg):
    m, img, ws, bgc, code, lm = _sr_inputs(part)
    bg_color = _bg(bg, ws.shape[0])
    res = m.torso_pass(img, ws, bgc, None, code(), bg_color=bg_color, lm68=lm)
    ref = composed_sr(m, img, ws, bgc, code(), bg_color, lm)
    print(f"\n[SR part {part}, {bg}] M = {ref['deform'].shape[0]} of {ws.shape[0]}")
    assert ref["deform"].shape[0] > 0
    _assert_equal_maps(res, ref)


# ------------------------------------------------------------------------------------------------ 3. golden (b)
def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def test_golden_b_with_frozen_head_and_torso_pass(golden):
    """frozen_head (fp32) + torso_pass + the task loss meet golden (b): maps within STEP_OUT; each weight and code gradient no further
    from float64 than max(2 x the reference's own fp32 error, FLOOR); the sampled table entries likewise and the table's per-level
    norms within max(2 x the reference's, 1e-4) of float64's."""
    m = golden["m"]
    z = np.load(GOLDEN)
    inp = {k: torch.from_numpy(z[f"b.{k}"]).cuda() for k in ("rays_o", "rays_d", "cond", "bg_coords", "bg_color", "gt")}
    index = torch.tensor([tt.GOLDEN_INDEX], device="cuda")
    m.zero_grad(set_to_none=True)
    with torch.no_grad():
        feat = m.cal_cond_feat(inp["cond"])
    ws, img = m.frozen_head(inp["rays_o"].reshape(-1, 3), inp["rays_d"].reshape(-1, 3), feat, m.individual_embeddings[index],
                            max_steps=tt.GOLDEN_MAX_STEPS)
    res = m.torso_pass(img, ws, inp["bg_coords"], torch.from_numpy(z["pose6"]).cuda(), m.torso_individual_codes[index], bg_color=inp["bg_color"])
    tt.task_loss(res, inp["gt"], tt.LAMBDA_WEIGHTS_ENTROPY).backward()
    torch.cuda.synchronize()
    for k in ("torso_alpha_map", "torso_rgb_map", "rgb_map", "weights_sum"):
        e = _rel(res[k].detach().reshape(-1), z[f"b.{k}"].reshape(-1))
        print(f"golden (b) {k}: rel {e:.2e}")
        assert e <= STEP_OUT, (k, e)
    params = dict(m.named_parameters())
    assert all(p.grad is None for k, p in params.items() if k not in tt.TRAINABLE + ["torso_individual_codes"]), "the head must stay frozen"
    gg = {k: params[k].grad.cpu() for k in tt.TRAINABLE}
    gg["code"] = params["torso_individual_codes"].grad[tt.GOLDEN_INDEX].cpu()
    for k in tt.TRAINABLE[:6] + ["code"]:
        e = _rel(gg[k], z[f"b.grad64.{k}"])
        e_ref = _rel(z[f"b.grad.{k}"], z[f"b.grad64.{k}"])
        print(f"golden (b) {k}: to float64 {e:.2e}, reference {e_ref:.2e}")
        assert e <= max(2 * e_ref, FLOOR), (k, e, e_ref)
    tab = gg["torso_embedder.embeddings"]
    e = _rel(tab[torch.from_numpy(z["table_sample_idx"])], z["b.grad64.table_sample"])
    e_ref = _rel(z["b.grad.table_sample"], z["b.grad64.table_sample"])
    off = golden["sc"].state["torso_embedder.offsets"].tolist()
    norms = np.asarray([float(tab[off[l]:off[l + 1]].double().norm()) for l in range(len(off) - 1)])
    n64 = np.maximum(z["b.grad64.table_level_norms"], 1e-30)
    en = float(np.max(np.abs(norms - n64) / n64))
    en_ref = float(np.max(np.abs(z["b.grad.table_level_norms"] - n64) / n64))
    print(f"golden (b) table: sampled {e:.2e} (reference {e_ref:.2e}); level norms {en:.2e} (reference {en_ref:.2e})")
    assert e <= max(2 * e_ref, FLOOR) and en <= max(2 * en_ref, 1e-4), (e, e_ref, en, en_ref)
    m.zero_grad(set_to_none=True)


# ------------------------------------------------------------------------------------------------ 4. gradients against the composed recipe
def _task_loss(res, gt, mode, deform_term):
    """torso_train_mode 1: MSE on torso_rgb_map; 0: MSE on rgb_map; both + the alpha entropy; the SR task adds lambda_torso_deform
    times mean |deform|."""
    key = "torso_rgb_map" if mode == 1 else "rgb_map"
    loss = ((res[key] - gt) ** 2).mean()
    a = res["torso_alpha_map"].clamp(1e-5, 1 - 1e-5)
    loss = loss + tt.LAMBDA_WEIGHTS_ENTROPY * (-a * torch.log2(a) - (1 - a) * torch.log2(1 - a)).mean()
    if deform_term:
        loss = loss + LAMBDA_DEFORM * res["deform"].abs().mean()
    return loss


def _clamp_edges(image, ws, trgb, mask):
    """image / weights_sum with some masked pixels' pre-clamp rgb_map exactly 0 (image = -t) or 1 (image = 1 - t), ws = 0."""
    image, ws = image.clone(), ws.clone()
    mi = mask.nonzero().reshape(-1)
    lo, hi = mi[0::7], mi[3::7]
    ws[lo], ws[hi] = 0, 0
    image[lo] = -trgb[lo]
    image[hi] = 1 - trgb[hi]
    x = image + (1 - ws).unsqueeze(-1) * trgb
    return image, ws, int((x == 0).sum()), int((x == 1).sum())


def _grads(m, names):
    params = dict(m.named_parameters())
    return {k: params[k].grad.detach().clone() for k in names}


@pytest.mark.parametrize("mode", [1, 0])
def test_torso_gradients_against_composed(golden, mode):
    s = golden
    m = s["m"]
    code = (lambda: m.torso_individual_codes[s["index"]])     # a fresh index node per graph
    bgc = s["fi"]["bg_color"].cuda()
    N = s["bg_coords"].shape[0]
    gt = tt.golden_target(N).cuda()
    with torch.no_grad():
        ref0 = composed_torso(m, s["img"], s["ws"], s["bg_coords"], s["pose6"], code(), bgc)
    img, ws, n0, n1 = _clamp_edges(s["img"], s["ws"], ref0["torso_rgb_map"], m.torso_mask(s["bg_coords"]))
    assert n0 > 0 and n1 > 0
    names = tt.TRAINABLE + ["torso_individual_codes"]
    m.zero_grad(set_to_none=True)
    _task_loss(composed_torso(m, img, ws, s["bg_coords"], s["pose6"], code(), bgc), gt, mode, False).backward()
    g_ref = _grads(m, names)
    m.zero_grad(set_to_none=True)
    _task_loss(m.torso_pass(img, ws, s["bg_coords"], s["pose6"], code(), bg_color=bgc), gt, mode, False).backward()
    g = _grads(m, names)
    m.zero_grad(set_to_none=True)
    print(f"\n[torso_train_mode {mode}] pre-clamp rgb_map exactly 0 at {n0} and 1 at {n1} channel(s)")
    for k in names:
        e = (g[k] - g_ref[k]).abs().max().item() / g_ref[k].abs().max().item()
        print(f"  {k}: {e:.2e} of max|grad|")
        assert e <= GRAD_REL, (k, e)


@pytest.mark.parametrize("part", ["b", "c"])
@pytest.mark.parametrize("mode", [1, 0])
def test_sr_gradients_against_composed(part, mode):
    m, img, ws, bgc, code, lm = _sr_inputs(part)
    bg_color = _bg("per_pixel", ws.shape[0])
    gt = tt.golden_target(ws.shape[0]).cuda()
    with torch.no_grad():
        ref0 = composed_sr(m, img, ws, bgc, code(), bg_color, lm)
    G = m.grid_size
    occ = F.grid_sample(m.density_grid_torso.view(1, 1, G, G), bgc.view(1, -1, 1, 2), align_corners=True).view(-1)
    img, ws, n0, n1 = _clamp_edges(img, ws, ref0["torso_rgb_map"], occ > min(m.density_thresh_torso, m.mean_density_torso))
    assert n0 > 0 and n1 > 0
    names = [k for k, p in m.named_parameters() if k.startswith(("torso_", "head_color_weights_encoder"))]
    m.zero_grad(set_to_none=True)
    _task_loss(composed_sr(m, img, ws, bgc, code(), bg_color, lm), gt, mode, True).backward()
    g_ref = _grads(m, names)
    m.zero_grad(set_to_none=True)
    _task_loss(m.torso_pass(img, ws, bgc, None, code(), bg_color=bg_color, lm68=lm), gt, mode, True).backward()
    g = _grads(m, names)
    print(f"\n[SR part {part}, torso_train_mode {mode}] pre-clamp exactly 0 at {n0}, 1 at {n1}")
    assert all(p.grad is None for k, p in m.named_parameters() if k not in names)
    for k in names:
        e = (g[k] - g_ref[k]).abs().max().item() / g_ref[k].abs().max().item()
        print(f"  {k}: {e:.2e} of max|grad|")
        assert e <= GRAD_REL, (k, e)


# ------------------------------------------------------------------------------------------------ 5. three Adam steps at step scale
@pytest.mark.parametrize("cls", ["torso", "sr"])
def test_adam_steps_at_step_scale(cls):
    """65 536 rays of a scene.Scene torso frame, the fp16 frozen head under autocast with a GradScaler (the torso configs' amp: true):
    three Adam steps of torso_pass and of the composed recipe from the same state."""
    sc = scn.Scene(H=256, W=256, T=4, torso=True, density_scale=tt.GOLDEN_DS)
    fi = sc.frame_inputs(1)
    ro, rd = fi["rays_o"].cuda().reshape(-1, 3), fi["rays_d"].cuda().reshape(-1, 3)
    bgc, bg_color = fi["bg_coords"].cuda().reshape(-1, 2), fi["bg_color"].cuda()
    N = ro.shape[0]
    gt = tt.golden_target(N).cuda()
    idx = torch.tensor([1], device="cuda")
    legs = []
    for _ in range(2):
        m = _torso(sc) if cls == "torso" else _sr("b", sc)
        m.mlp_precision = "fp16"
        names = [k for k, p in m.named_parameters() if k.startswith(("torso_", "head_color_weights_encoder"))]
        ps = [p for k, p in m.named_parameters() if k in names]
        legs.append((m, ps, torch.optim.Adam(ps, lr=1e-3 if cls == "torso" else 5e-3), torch.amp.GradScaler("cuda")))
    if cls == "torso":
        cond = fi["cond"].cuda()
        feat_kw = {}
    else:
        cond = scn.cond_window(sc.cond, 1, legs[0][0].hparams["smo_win_size"]).cuda()
        feat_kw = {"eye_area_percent": torch.tensor([0.3], device="cuda")}
    lm = tst.golden_lm68().cuda()
    losses = [[], []]
    for it in range(4):
        for leg, (m, ps, opt, scaler) in enumerate(legs):
            opt.zero_grad()
            with torch.autocast("cuda", dtype=torch.float16):
                with torch.no_grad():
                    feat = m.cal_cond_feat(cond, **feat_kw)
                ws, img = m.frozen_head(ro, rd, feat, m.individual_embeddings[idx], max_steps=16)
                code = m.torso_individual_codes[idx]
                if leg == 0:
                    res = m.torso_pass(img, ws, bgc, fi["poses"].cuda(), code, bg_color=bg_color, lm68=lm)
                elif cls == "torso":
                    res = composed_torso(m, img, ws, bgc, fi["poses"].cuda(), code, bg_color)
                else:
                    res = composed_sr(m, img, ws, bgc, code, bg_color, lm)
                loss = _task_loss(res, gt, 1, cls == "sr")
            losses[leg].append(loss.item())
            if it < 3:
                scaler.scale(loss).backward()
                scaler.step(opt)
                scaler.update()
    la, lb = losses
    dl = max(abs(a - b) / abs(b) for a, b in zip(la, lb))
    dp = max((a.detach() - b.detach()).norm().item() / b.detach().norm().item() for a, b in zip(legs[0][1], legs[1][1]))
    print(f"\n[{cls}] M = {res['deform'].shape[0]} of {N}; Adam x3: loss {la[0]:.6f} -> {la[-1]:.6f}; max rel loss diff {dl:.2e}; "
          f"max rel L2 param diff {dp:.2e}")
    assert la[-1] < la[0]
    assert dl <= ADAM_LOSS_REL and dp <= ADAM_PARAM_REL, (dl, dp)


# ------------------------------------------------------------------------------------------------ 6. determinism and M == 0
def test_determinism_and_empty_mask(golden):
    s = golden
    m = s["m"]
    bgc = s["fi"]["bg_color"].cuda()
    gt = tt.golden_target(s["bg_coords"].shape[0]).cuda()
    names = tt.TRAINABLE + ["torso_individual_codes"]
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        res = m.torso_pass(s["img"], s["ws"], s["bg_coords"], s["pose6"], m.torso_individual_codes[s["index"]], bg_color=bgc)
        _task_loss(res, gt, 0, False).backward()
        runs.append(({k: v.detach().clone() for k, v in res.items()}, _grads(m, names)))
    (r1, g1), (r2, g2) = runs
    for k in r1:
        assert torch.equal(r1[k], r2[k]), k
    for k in names:
        if k != "torso_embedder.embeddings":        # scattered with vector reductions: summation order free
            assert torch.equal(g1[k], g2[k]), k
    m.zero_grad(set_to_none=True)
    saved, thr = m.mean_density_torso, m.density_thresh_torso
    try:
        m.mean_density_torso = m.density_thresh_torso = 2.0     # above every occupancy of the 0 / 1 grid
        code = m.torso_individual_codes[s["index"]]
        res = m.torso_pass(s["img"], s["ws"], s["bg_coords"], s["pose6"], code, bg_color=bgc)
        assert m.last_launch_count == 3 + 1          # the mask and the composite: no field launch
        ref = composed_torso(m, s["img"], s["ws"], s["bg_coords"], s["pose6"], code, bgc)
        assert "deform" not in res and "deform" not in ref
        _assert_equal_maps(res, ref, ("torso_alpha_map", "torso_rgb_map", "rgb_map"))
        assert not any(v.requires_grad for v in res.values())
        assert int(res["torso_alpha_map"].count_nonzero()) == 0
        assert all(p.grad is None for k, p in m.named_parameters() if k in names)
    finally:
        m.mean_density_torso, m.density_thresh_torso = saved, thr
