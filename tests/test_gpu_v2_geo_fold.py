"""Sigma L2's geo rows folded into color L0 in the row-owner head kernel (k_head_v2, DESIGN §5): the fp16 and robust modes never
form the 128 geo features, color L0 runs W_fold = W_c0[:, 16:144] . W_s2[1:129, :] over sigma L1's output.

Scaling sigma L2's geo rows by 2^s and color L0's geo columns by 2^-s leaves the field unchanged and W_fold bit-identical (power-of-two
scaling is exact), while the geo features themselves grow past the fp16 range.  A kernel that still rounded them to fp16 operands
would overflow; the folded kernel must render the scaled model bit for bit as the unscaled one, and both within 1e-3 of the oracle."""
import math

import pytest
import torch
import torch.nn.functional as F

from genefaceplusplus_b200 import scene as scn
from helpers import build_model, parity_report

pytestmark = pytest.mark.gpu
TOL = 1e-3
FP16_MAX = 65504.0
FRAME = 2
_REF = {}


def _oracle_and_geo_max(size):
    """The scene, the oracle's render of FRAME on the rays the kernel generates, and the largest |geo| its field produced."""
    if size not in _REF:
        from oracle.render import OracleModel
        sc = scn.Scene(H=size, W=size, T=8, torso=True, density_scale=8.0)
        ro, rd = build_model(sc, precision="fp32").generate_rays(sc.pose(FRAME).view(1, 4, 4), sc.intrinsics, size, size)
        orc = OracleModel(sc.state, sc.hparams)
        orc.density_scale = sc.density_scale
        w_s2, geo_max = orc.st["sigma_net.net.2.weight"], [0.0]

        def linear(x, w):
            y = F.linear(x, w)
            if w is w_s2 and y.numel():
                geo_max[0] = max(geo_max[0], y[..., 1:].abs().max().item())
            return y

        orc._linear = linear
        fi = sc.frame_inputs(FRAME)
        ref = orc.render(ro.cpu(), rd.cpu(), fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **sc.hparams)
        _REF[size] = (sc, ref, geo_max[0])
    return _REF[size]


def _clip(model, sc):
    feat = model.cal_cond_feat_clip(sc.cond.cuda())[[FRAME]]
    return model.render_clip(sc.pose(FRAME).view(1, 4, 4), sc.intrinsics, sc.H, sc.W, cond_feat=feat, bg_color=sc.bg_color,
                             bg_coords=sc.bg_coords, T_thresh=sc.T_thresh)[0].cpu()


@pytest.mark.parametrize("size", [64, 512])
@pytest.mark.parametrize("precision", ["fp16", "robust"])
def test_geo_features_beyond_fp16_range(oracle_ops, precision, size):
    sc, ref, geo_max = _oracle_and_geo_max(size)
    # 16x past the fp16 range at the largest |geo|, so that many samples' geo features would overflow, not just that one
    s = math.ceil(math.log2(FP16_MAX / geo_max)) + 4
    st = dict(sc.state)
    w_s2 = st["sigma_net.net.2.weight"].clone()
    w_c0 = st["color_net.net.0.weight"].clone()
    w_s2[1:129] *= 2.0 ** s
    w_c0[:, 16:144] *= 2.0 ** -s
    assert torch.equal(w_s2[1:129] * 2.0 ** -s, sc.state["sigma_net.net.2.weight"][1:129])
    assert torch.equal(w_c0[:, 16:144] * 2.0 ** s, sc.state["color_net.net.0.weight"][:, 16:144]), "the rescaling must be exact"
    st["sigma_net.net.2.weight"], st["color_net.net.0.weight"] = w_s2, w_c0
    base = _clip(build_model(sc, precision=precision), sc)
    scaled = _clip(build_model(sc, st, precision=precision), sc)
    rep = parity_report(scaled, ref["rgb_map"].view(-1, 3), ref["knife"])
    print(f"[geo fold {precision} {size}^2] max|geo| {geo_max:.3g} x 2^{s}; scaled == unscaled: {torch.equal(scaled, base)}; "
          f"rgb max|d| vs oracle {rep['max_abs']:.2e} (knife {rep['n_knife']}) psnr={rep['psnr']:.1f}")
    assert geo_max * 2.0 ** s > FP16_MAX
    assert torch.equal(scaled, base), "the rescaled model must render bit for bit as the unscaled one"
    assert rep["max_abs"] <= TOL and rep["psnr"] >= 50
