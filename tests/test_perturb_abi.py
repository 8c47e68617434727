"""perturb=True without a GPU: the C-ABI field that carries the jitter, and the CPU-model guard of all four classes."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.config import may_hparams
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso, RADNeRFTorsowithSR, RADNeRFwithSR


def test_frames_noises_is_the_last_field():
    names = [f[0] for f in _capi.Frames._fields_]
    assert names[-2:] == ["T_thresh", "noises"]
    assert _capi.Frames._fields_[-1][1] is ctypes.c_void_p
    # appended: every earlier field keeps its offset, and a zero-initialised struct means "no jitter"
    assert _capi.Frames.noises.offset >= _capi.Frames.T_thresh.offset + ctypes.sizeof(ctypes.c_float)
    assert _capi.Frames().noises is None


def test_header_declares_noises_last():
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gfpp.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} gfpp_frames;", hdr).group(1)
    fields = [ln.split("/*")[0].strip() for ln in body.splitlines()]
    fields = [f for f in fields if f]
    assert fields[-2:] == ["float T_thresh;", "const float *noises;"]


def _render(m, H, W, hp, **extra):
    sc = scn.Scene(H=H, W=W, T=2, torso=True)
    fi = sc.frame_inputs(0)
    return m.render(fi["rays_o"], fi["rays_d"], scn.cond_window(sc.cond, 0, hp["smo_win_size"]), fi["bg_coords"], fi["poses"], index=0,
                    staged=False, bg_color=fi["bg_color"], perturb=True, force_all_rays=False, T_thresh=0.01, **{**hp, **extra})


@pytest.mark.parametrize("cls", [RADNeRF, RADNeRFTorso, RADNeRFwithSR, RADNeRFTorsowithSR], ids=lambda c: c.__name__)
def test_cpu_model_with_perturb_has_no_cpu_path(cls):
    sr = cls in (RADNeRFwithSR, RADNeRFTorsowithSR)
    hp = may_hparams(with_sr=True) if sr else may_hparams()
    m = cls(hp).eval()
    extra = {"lm68": torch.zeros(1, 136)} if cls is RADNeRFTorsowithSR else {}
    R = 256 if sr else 8
    state = torch.get_rng_state()
    with pytest.raises(_capi.GfppError):
        _render(m, R, R, hp, **extra)
    # nothing was drawn before the model's device was checked
    assert torch.equal(state, torch.get_rng_state())
