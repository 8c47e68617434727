"""The SR head on libgfpp's own sm_90a kernels (csrc/sr_kernel.cu; SURVEY 8(f) rank 3) against
  (i)  oracle/sr_emulate.py -- the CPU emulation of the kernels' data flow with the same fp16 operand rounding.  The fp16
       activations the kernels keep in their workspace must equal the emulation's up to fp16 rounding flips (fp32 accumulation
       order decides a rounding tie differently now and then; on the H100: max 9.77e-4 = one fp16 ulp at |x| in [1,2) in the
       fp16 layers, 0.6 % of the second layer's elements affected), and the final image to 1e-3 (2.6-3.6e-4 on the H100: the
       effect of those flips).  A layout / descriptor / pipeline bug is O(1) on both;
  (ii) the fp32 convolutions of `Superresolution.forward` (pinned to the REFERENCE's Superresolution by tests/golden/sr_head.npz)
       and that golden itself: the 1e-3 bar on the clamped image the drivers consume."""
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.superres import Superresolution

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _net():
    g = np.load(os.path.join(GOLD, "sr_head.npz"))
    meta = json.loads(bytes(g["meta"]).decode())
    net = Superresolution(channels=3).eval()
    net.load_state_dict(scn.synthetic_sr_state({k: tuple(v) for k, v in meta["shapes"].items()}, seed=3), strict=False)
    return net, g, meta


def _inputs():
    full = scn.hashed_uniform(3 * 256 * 256, 78, 1.0).reshape(1, 3, 256, 256) + 0.5
    x = torch.cat([full, full.flip(-1), full.flip(-2) * 0.5], 0)          # 3 frames: frame indexing + borders differ
    return x, x.permute(0, 2, 3, 1).reshape(3, -1, 3).contiguous()


@pytest.mark.parametrize("mode", ["const", "none", "planes"])
def test_native_sr_head_matches_emulation_and_fp32(mode):
    from oracle.sr_emulate import emulate
    net, g, meta = _net()
    x, flat = _inputs()
    lay = net._layers()
    with torch.no_grad():
        if mode == "const":
            nz = [(l.noise_const * l.noise_strength).float() for l in lay]
            ref = net(x, noise_mode="const")
        elif mode == "none":
            nz = [None] * 4
            ref = net(x, noise_mode="none")
        else:   # one plane per frame (what noise_mode='random' hands the kernels), injected so that the checker sees the same
            gen = torch.Generator().manual_seed(5)
            nz = [torch.randn(3, l.resolution, l.resolution, generator=gen) * 0.05 for l in lay]
            ref = None
        inter = {}
        emu = emulate(net.folded_weights(), flat, 256, nz, fp16=True, intermediates=inter)
    net = net.cuda()
    net.backend = "native"
    got = net.forward_native(flat.cuda(), noise_mode="none" if mode == "none" else "const",
                             noise_planes=None if mode != "planes" else [p.cuda() for p in nz], frames_per_call=2)
    torch.cuda.synchronize()
    got = got.cpu()
    # layer-by-layer diagnosis from the kernels' workspace (last chunk of frames: frames_per_call=2 -> frame 2 only)
    ws, R, n_last = net.__dict__["_native"]["ws"], 256, 1
    px = n_last * R * R
    off, parts = 0, {}
    for name, numel, dt in (("x0a", px * 128, torch.float16), ("x0b", px * 128, torch.float16), ("img0", px * 3, torch.float32), ("x1a", px * 4 * 64, torch.float16)):
        nbytes = numel * (2 if dt == torch.float16 else 4)
        parts[name] = ws[off:off + nbytes].view(dt).float().cpu()
        off += (nbytes + 255) // 256 * 256
    for name, t in parts.items():
        ref_t = inter[name][2:3].reshape(-1)
        d = (t - ref_t).abs()
        off = (d > 0).float().mean().item()
        print(f"[{mode}] workspace {name}: |kernel - emulation| max {d.max().item():.3e}, mean {d.mean().item():.3e} (scale {ref_t.abs().max().item():.2f}), elements that differ: {off:.2e}")
        # x0a comes straight from the fp32 input layer: identical up to one fp16 ulp (2^-10 at |x| in [1,2)) on ~3e-4 of the elements.
        # Downstream an input that moved by an ulp shifts a sum by ~1e-4, which re-rounds many small outputs by their (tiny) ulp:
        # the count of differing elements is meaningless there, the size of the difference is not.
        assert d.max().item() <= (2e-3 if name == "x0a" else 4e-3 if name != "img0" else 3e-4) and d.mean().item() <= 3e-4, name
        if name == "x0a":
            assert off <= 5e-3, name
    assert torch.isfinite(got).all()
    e_model = (got - emu).abs().max().item()
    print(f"[{mode}] |native - fp16 data-flow emulation| = {e_model:.3e}")
    assert e_model <= 1e-3, "layout / descriptor / pipeline error (not a rounding effect)"
    if ref is not None:
        e32 = (got.clamp(0, 1) - ref.clamp(0, 1)).abs().max().item()
        psnr = 10 * np.log10(1.0 / max((got.clamp(0, 1) - ref.clamp(0, 1)).square().mean().item(), 1e-20))
        print(f"[{mode}] |native - fp32 convolutions| on the clamped image = {e32:.3e}, PSNR {psnr:.1f} dB")
        assert e32 <= 1e-3 and psnr >= 50.0
    if mode == "const":   # frame 0 is the golden's input: the reference's own Superresolution output
        c0, c1, c2, c3 = meta["crop"]
        crop = torch.from_numpy(g["in256_crop"])
        eg = (got[0, :, c0:c1, c2:c3].clamp(0, 1) - crop.clamp(0, 1)).abs().max().item()
        print(f"[const] |native - reference golden crop| = {eg:.3e}")
        assert eg <= 1e-3
        # forward() routes CUDA tensors to the same kernels; clamp flag of the last epilogue
        y = net(x[:1].cuda(), noise_mode="const").cpu()
        assert (y - got[:1]).abs().max().item() == 0.0
        yc = net.forward_native(flat[:1].cuda(), noise_mode="const", clamp=True).cpu()
        assert (yc - got[:1].clamp(0, 1)).abs().max().item() == 0.0


def test_native_sr_repacks_when_a_parameter_changes():
    net, _, _ = _net()
    _, flat = _inputs()
    net = net.cuda()
    net.backend = "native"
    a = net.forward_native(flat[:1].cuda(), noise_mode="none").clone()
    with torch.no_grad():
        net.block1.conv1.bias.add_(0.25)
    b = net.forward_native(flat[:1].cuda(), noise_mode="none")
    torch.cuda.synchronize()
    assert (a - b).abs().max().item() > 1e-3


# ------------------------------------------------------------------------------------------------ torso-SR field in libgfpp
def _torso_sr(head_aware):
    from genefaceplusplus_b200.config import may_hparams
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
    z = np.load(os.path.join(GOLD, "torso_sr256.npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    hp = may_hparams(**{**meta["overrides"], "torso_head_aware": head_aware})
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    m = m.cuda().eval()
    sc = scn.Scene(H=256, W=256, T=8, torso=True, density_scale=meta["density_scale"])
    return m, hp, sc, z, meta


def _render(m, hp, sc, meta, t, **extra):
    fi = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in sc.frame_inputs(t).items()}
    lm68 = scn.lm68_sequence(8)[t].reshape(1, 136).cuda()
    kw = {k: v for k, v in hp.items() if k not in ("max_steps", "dt_gamma")}
    return m.render(fi["rays_o"], fi["rays_d"], scn.cond_window(sc.cond, t, 3).cuda(), fi["bg_coords"], fi["poses"], index=t,
                    dt_gamma=hp["dt_gamma"], bg_color=fi["bg_color"], max_steps=16, T_thresh=sc.T_thresh, upscale_torso=True, lm68=lm68,
                    eye_area_percent=torch.tensor([[meta["eye"]]]), sr_noise_mode="const", **kw, **extra)


@pytest.mark.parametrize("head_aware", [True, False])
def test_torso_sr_field_native_matches_the_host_path(head_aware):
    """k_torso_sr (libgfpp) against the host-side torch field over the per-op encoder kernels -- itself pinned to the reference's
    render() golden (tests/test_gpu_sr.py) -- on the same head image: fp32 both, so 2e-5 on every 256x256 map (H100:
    <= 1.1e-6).  `sr_rgb_map` goes through the host-side cuDNN convolutions here (TF32): two runs on inputs 5e-7 apart differ by
    ~4e-4 there, so it only gets the 1e-3 bar."""
    m, hp, sc, z, meta = _torso_sr(head_aware)
    m.sr_net.backend = "torch"
    t = meta["frame"]
    m.torso_backend = "torch"
    ref = _render(m, hp, sc, meta, t)
    m.torso_backend = "native"
    got = _render(m, hp, sc, meta, t)
    torch.cuda.synchronize()
    for k in ("rgb_map", "torso_rgb_map", "torso_alpha_map", "deform", "sr_rgb_map"):
        e = (got[k].float() - ref[k].float()).abs().max().item()
        print(f"head_aware={head_aware} {k}: |native - host| = {e:.3e}")
        assert got[k].shape == ref[k].shape and e <= (2e-5 if k != "sr_rgb_map" else 1e-3), (k, e)
    if head_aware:   # the golden was made with torso_head_aware=True: the reference's own render()
        for k, (a, b, c, d) in meta["crops"].items():
            e = (got[k][0, :, a:b, c:d].float().cpu() - torch.from_numpy(z[f"{k}_crop"])).abs().max().item()
            print(f"{k}: |native - reference golden| = {e:.3e}")
            assert e <= 1e-3, (k, e)
        assert abs(got["torso_alpha_map"].double().sum().item() - float(z["torso_alpha_sum"][0])) < 1.0


def test_torso_sr_clip_all_native_matches_per_frame_render():
    """render_clip with every stage in libgfpp (head field with in-kernel rays, torso-SR field, SR head) against per-frame
    render() with the host-side torso field and fp32 SR convolutions."""
    m, hp, sc, z, meta = _torso_sr(True)
    T = 3
    m.torso_backend, m.sr_net.backend = "torch", "torch"
    ref = torch.stack([_render(m, hp, sc, meta, t)["sr_rgb_map"][0] for t in range(T)])
    m.torso_backend, m.sr_net.backend = "native", "native"
    poses = torch.stack([sc.pose(t) for t in range(T)]).cuda()
    eye = torch.full((8,), meta["eye"])   # conditioning of the whole 8-frame sequence: same windows as cond_window(sc.cond, t, 3)
    got = m.render_clip(poses, sc.intrinsics, 256, 256, cond_seq=sc.cond.cuda(), bg_color=sc.bg_color.cuda(), bg_coords=sc.bg_coords.cuda(),
                        lm68_seq=scn.lm68_sequence(8)[:T].cuda(), eye_area_percent=eye, max_steps=16, T_thresh=sc.T_thresh, sr_noise_mode="const",
                        frames_per_call=2)
    torch.cuda.synchronize()
    d = (got - ref).abs()
    frac = (d > 1e-3).float().mean().item()   # in-kernel rays differ from get_rays by <= 2 ulp: rare occupancy-cell flips (DESIGN 6)
    psnr = 10 * np.log10(1.0 / max(d.square().mean().item(), 1e-20))
    print(f"torso-SR clip, all native: max {d.max().item():.3e}, fraction > 1e-3: {frac:.2e}, PSNR {psnr:.1f} dB")
    assert frac <= 1e-4 and psnr >= 50.0
