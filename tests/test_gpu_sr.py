"""GPU runs of the SR-variant drop-ins (SURVEY 8(f) rank 3) against the reference goldens: `RADNeRFwithSR` / `RADNeRFTorsowithSR`
with the head field in libgfpp's fused kernels at 256x256 and the SR head (and, for the torso-SR variant, its torso field and
composite) as host-side PyTorch over libgfpp's per-op encoder kernels.
The CPU halves of these checks run in tests/test_host_logic.py and tests/test_oracle_golden.py."""
import json
import os

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _load(name):
    z = np.load(os.path.join(GOLD, name))
    return z, json.loads(bytes(z["meta"]).decode())


def _check(out, z, meta, tol):
    for k, (a, b, c, d) in meta["crops"].items():
        got = out[k][0, :, a:b, c:d].float().cpu()
        ref = torch.from_numpy(z[f"{k}_crop"])
        err = (got - ref).abs().max().item()
        psnr = 10 * np.log10(1.0 / max((got - ref).square().mean().item(), 1e-20))
        print(f"{k}: max|gpu - reference| = {err:.3e}, PSNR {psnr:.1f} dB")
        assert err <= tol and psnr >= 50.0, (k, err, psnr)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_head_sr_model_on_gpu(precision):
    from genefaceplusplus_b200.renderer import RADNeRFwithSR
    z, meta = _load("head_sr256.npz")
    hp = may_hparams(**meta["overrides"])
    m = RADNeRFwithSR(hp)
    m.load_state_dict(scn.make_head_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    m.mlp_precision = precision
    m = m.cuda().eval()
    sc = scn.Scene(H=256, W=256, T=8, torso=False, density_scale=meta["density_scale"])
    t = meta["frame"]
    fi = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in sc.frame_inputs(t).items()}
    kw = {k: v for k, v in hp.items() if k not in ("max_steps", "dt_gamma")}
    out = m.render(fi["rays_o"], fi["rays_d"], scn.cond_window(sc.cond, t, 3).cuda(), fi["bg_coords"], fi["poses"], index=t,
                   dt_gamma=hp["dt_gamma"], bg_color=fi["bg_color"], max_steps=16, T_thresh=sc.T_thresh,
                   eye_area_percent=torch.tensor([[meta["eye"]]]), **kw)
    _check(out, z, meta, 1e-3)


def test_torso_sr_model_on_gpu():
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR
    z, meta = _load("torso_sr256.npz")
    hp = may_hparams(**meta["overrides"])
    m = RADNeRFTorsowithSR(hp)
    m.load_state_dict(scn.make_torso_sr_state(hp), strict=True)
    m.density_scale = meta["density_scale"]
    m = m.cuda().eval()
    sc = scn.Scene(H=256, W=256, T=8, torso=True, density_scale=meta["density_scale"])
    t = meta["frame"]
    fi = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in sc.frame_inputs(t).items()}
    lm68 = scn.lm68_sequence(8)[t].reshape(1, 136).cuda()
    kw = {k: v for k, v in hp.items() if k not in ("max_steps", "dt_gamma")}
    out = m.render(fi["rays_o"], fi["rays_d"], scn.cond_window(sc.cond, t, 3).cuda(), fi["bg_coords"], fi["poses"], index=t,
                   dt_gamma=hp["dt_gamma"], bg_color=fi["bg_color"], max_steps=16, T_thresh=sc.T_thresh, upscale_torso=True, lm68=lm68,
                   eye_area_percent=torch.tensor([[meta["eye"]]]), **kw)
    _check(out, z, meta, 1e-3)
    assert abs(out["torso_alpha_map"].double().sum().item() - float(z["torso_alpha_sum"][0])) < 1.0
