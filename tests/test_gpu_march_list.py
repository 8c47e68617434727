"""Pass-1 sample lists of the row-owner head kernel (k_march_list + k_head_v2, DESIGN §5): k_march_list marches every hit ray's
samples 2 .. 16 ahead of pass 1 and the row owners rebuild each sample from its stored pre-step t with sample_at; past a full list
(max_steps > 16) and in pass 2 they march as before.  Every march step is a pure function of t, so the lists must not change a bit:
each call is rendered with the lists (the default) and with GFPP_MARCH_LIST=0, which keeps the march in the owners, and every map
and B / S / P must be equal, in both modes of the kernel, at sample caps on both sides of the list length, with jittered starts,
multi-frame calls, the bench's 50-frame 512^2 call and a scene that sends rays to pass 2."""
import pytest
import torch

from genefaceplusplus_b200 import scene as scn
from helpers import build_model

pytestmark = pytest.mark.gpu
MAPS = ("rgb_map", "depth_map", "weights_sum", "torso_alpha_map", "torso_rgb_map", "deform")
PRECISIONS = ("fp16", "robust")


def _same(a, b):
    """torch.equal, NaN positions (the depth of rays that miss the aabb) included."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.masked_fill(na, 0.0), b.masked_fill(nb, 0.0))


def _both(monkeypatch, fn):
    """fn() with the sample lists on, then off."""
    monkeypatch.delenv("GFPP_MARCH_LIST", raising=False)
    on = fn()
    monkeypatch.setenv("GFPP_MARCH_LIST", "0")
    off = fn()
    monkeypatch.delenv("GFPP_MARCH_LIST", raising=False)
    return on, off


def _render_both(monkeypatch, sc, prec, frames, max_steps, T_thresh, noise=None, rays=None):
    model = build_model(sc, precision=prec)
    feat = model.cal_cond_feat_clip(sc.cond.cuda())[list(frames)]
    poses = torch.stack([sc.pose(t) for t in frames])
    kw = dict(pose6=scn.convert_poses(poses).cuda(), bg_coords=sc.bg_coords.cuda(), bg_color=sc.bg_color.cuda(),
              dt_gamma=sc.hparams["dt_gamma"], max_steps=max_steps, T_thresh=T_thresh, noise=noise, want_stats=True)
    if rays is None:
        kw.update(poses_c2w=poses.cuda(), intrinsics=sc.intrinsics, H=sc.H, W=sc.W)
    else:
        kw.update(rays_o=rays[0].cuda(), rays_d=rays[1].cuda())
    on, off = _both(monkeypatch, lambda: model.render_frames(feat, **kw))
    bad = [k for k in MAPS if k in on and not _same(on[k], off[k])]
    st_on, st_off = on["stats"].cpu(), off["stats"].cpu()
    print(f"[march list, {prec}] F={len(frames)} max_steps {max_steps} T_thresh {T_thresh}: maps differing {bad}; "
          f"B {int(st_on[0, 0])} S {int(st_on[:, 2].sum())} survivors {int(st_on[0, 1])}")
    assert not bad and torch.equal(st_on, st_off)
    return st_on


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("max_steps", [1, 8, 16, 17, 32])
@pytest.mark.parametrize("T_thresh", [1e-4, 1e-2])
@pytest.mark.parametrize("perturb", [False, True])
def test_render_equal_without_lists(monkeypatch, prec, max_steps, T_thresh, perturb):
    sc = scn.Scene(H=128, W=128, T=3, torso=True, density_scale=8.0)
    frames = [0, 1, 2]
    noise = (torch.rand(len(frames), sc.H * sc.W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
             if perturb else None)
    _render_both(monkeypatch, sc, prec, frames, max_steps, T_thresh, noise=noise)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_bench_call_equal_without_lists(monkeypatch, prec):
    sc = scn.Scene(H=512, W=512, T=50, torso=True, density_scale=8.0)
    _render_both(monkeypatch, sc, prec, list(range(50)), 16, 0.01)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_pass2_equal_without_lists(monkeypatch, prec):
    # translucent scene, as test_gpu_v2_gather_warps.py::test_pass2_50x50_max_steps_8: rays outlive pass 1's cap and pass 2 marches on
    sc = scn.Scene(H=50, W=50, T=8, torso=True, max_steps=8, density_scale=1.0)
    frames = list(range(8))
    rays = (torch.cat([sc.frame_inputs(t)["rays_o"] for t in frames]), torch.cat([sc.frame_inputs(t)["rays_d"] for t in frames]))
    st = _render_both(monkeypatch, sc, prec, frames, 8, sc.T_thresh, rays=rays)
    assert int(st[0, 1]) > 0, "rays must reach pass 2"
