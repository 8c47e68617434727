"""The frozen head's C-ABI (gfpp.h section K) and RADNeRF.frozen_head's guards, without a GPU: every argument is validated before
any CUDA call (a CUDA call on this machine would return GFPP_ERR_CUDA instead of the codes checked here)."""
import ctypes

import pytest
import torch

from genefaceplusplus_b200 import _capi
from genefaceplusplus_b200 import scene as scn
from genefaceplusplus_b200.renderer import RADNeRF, RADNeRFTorso

OK, INVALID, WORKSPACE, UNSUPPORTED = 0, -1, -3, -4
FAKE = 0x10000          # 256-byte aligned, never dereferenced: validation fails first
MAGIC = 0x67667070      # the first word of a handle filled by gfpp_model_pack


@pytest.fixture(scope="module")
def L():
    from genefaceplusplus_b200 import build
    build.build()
    return _capi.lib()


def _handle():
    """A gfpp_model handle that passes the handle check (magic word set) and describes a model without individual codes."""
    m = _capi.Model()
    m.opaque[0] = MAGIC
    return m


AABB = (ctypes.c_float * 6)(-1, -0.5, -1, 1, 0.5, 1)


def _call(L, model=True, ro=FAKE, rd=FAKE, N=1024, aabb=AABB, cond=FAKE, code=None, noises=None, max_steps=16, ws=None, ws_ptr=FAKE,
          wsum=FAKE, image=FAKE, m=None):
    ws_bytes = L.gfpp_frozen_head_workspace_bytes(max(N, 1), max_steps if 1 <= max_steps <= 4096 else 16) if ws is None else ws
    h = m if m is not None else _handle()
    return L.gfpp_frozen_head(ctypes.byref(h) if model else None, ro, rd, N, aabb, cond, code, noises, 0.0, max_steps, 1e-4, wsum, image,
                              ws_ptr, ws_bytes, None)


def test_symbols_and_workspace_sizes(L):
    for n in ("gfpp_frozen_head_workspace_bytes", "gfpp_frozen_head"):
        assert n in _capi.EXPORTS and hasattr(L, n)
    assert L.gfpp_frozen_head_workspace_bytes(0, 16) == 0
    assert L.gfpp_frozen_head_workspace_bytes(1 << 31, 16) == 0
    assert L.gfpp_frozen_head_workspace_bytes(1024, 0) == 0
    assert L.gfpp_frozen_head_workspace_bytes(1024, 4097) == 0
    sizes = [L.gfpp_frozen_head_workspace_bytes(N, 16) for N in (1, 1024, 65536, 1 << 20)]
    assert all(s % 256 == 0 for s in sizes) and sizes == sorted(sizes) and sizes[0] < sizes[-1]
    # the per-ray part: depth, resume t, survivor id (4 B each) and a 64-byte hit record
    assert sizes[3] - sizes[2] == ((1 << 20) - 65536) * 76
    assert L.gfpp_frozen_head_workspace_bytes(1024, 4096) > L.gfpp_frozen_head_workspace_bytes(1024, 16)


def test_null_pointers(L):
    assert _call(L, model=False) == INVALID
    for kw in ({"ro": None}, {"rd": None}, {"aabb": None}, {"cond": None}, {"wsum": None}, {"image": None}, {"ws_ptr": None}):
        assert _call(L, **kw) == INVALID, kw
        assert b"null pointer" in L.gfpp_last_error()


def test_handle_not_packed(L):
    assert _call(L, m=_capi.Model()) == INVALID
    assert b"gfpp_model_pack" in L.gfpp_last_error()


def test_sizes(L):
    assert _call(L, N=0) == INVALID
    assert b"no rays" in L.gfpp_last_error()
    assert _call(L, N=1 << 31, ws=1 << 40) == UNSUPPORTED
    assert _call(L, max_steps=0) == UNSUPPORTED
    assert _call(L, max_steps=4097) == UNSUPPORTED


def test_code_iff_ind_dim(L):
    # a model packed without individual codes takes no code
    assert _call(L, code=FAKE) == INVALID
    assert b"code must be given iff" in L.gfpp_last_error()


def test_aabb_order(L):
    bad = (ctypes.c_float * 6)(1, -0.5, -1, -1, 0.5, 1)
    assert _call(L, aabb=bad) == INVALID
    nan = (ctypes.c_float * 6)(float("nan"), -0.5, -1, 1, 0.5, 1)
    assert _call(L, aabb=nan) == INVALID


def test_workspace(L):
    need = L.gfpp_frozen_head_workspace_bytes(1024, 16)
    assert _call(L, ws=need - 1) == WORKSPACE
    assert b"workspace too small" in L.gfpp_last_error()
    assert _call(L, ws_ptr=FAKE + 16) == INVALID
    assert b"256-byte aligned" in L.gfpp_last_error()


# ------------------------------------------------------------------------------------------------ RADNeRF.frozen_head
def _torso_model():
    sc = scn.Scene(H=8, W=8, T=2, torso=True)
    m = RADNeRFTorso(sc.hparams)
    m.load_state_dict(sc.state, strict=True)
    return m


def test_every_class_has_frozen_head():
    from genefaceplusplus_b200.renderer import RADNeRFTorsowithSR, RADNeRFwithSR
    for cls in (RADNeRF, RADNeRFwithSR, RADNeRFTorso, RADNeRFTorsowithSR):
        assert cls.frozen_head is RADNeRF.frozen_head


def test_cpu_model_raises():
    m = _torso_model()
    ro, rd = torch.zeros(4, 3), torch.ones(4, 3)
    with pytest.raises(_capi.GfppNoCpuPath):
        m.frozen_head(ro, rd, torch.zeros(64), m.individual_embeddings[0])
    m.train()
    with pytest.raises(_capi.GfppNoCpuPath):
        m.frozen_head(ro, rd, torch.zeros(64), m.individual_embeddings[0], perturb=True)


def _guard(m, **kw):
    """Calls frozen_head with the device check passed (density_bitfield stands in for a CUDA tensor) and returns what it raised."""
    args = dict(rays_o=torch.zeros(4, 3), rays_d=torch.ones(4, 3), cond_feat=torch.zeros(64), ind_code=m.individual_embeddings[0])
    args.update(kw)
    orig = m._buffers["density_bitfield"]
    try:
        m._buffers["density_bitfield"] = _FakeCuda(orig)
        with pytest.raises(Exception) as e:
            m.frozen_head(**args)
        return e.value
    finally:
        m._buffers["density_bitfield"] = orig


class _FakeCuda:
    """Stands in for density_bitfield: reports a CUDA device, and anything beyond the guards fails loudly."""

    def __init__(self, t):
        self.t = t

    @property
    def device(self):
        return torch.device("cuda", 0)

    def __getattr__(self, k):
        raise AssertionError(f"frozen_head went past its guards (touched density_bitfield.{k})")


def test_mean_count_guard():
    m = _torso_model()
    m.mean_count = 1000
    e = _guard(m)
    assert isinstance(e, ValueError) and "mean_count" in str(e)
    # force_all_rays lifts it: the call then goes past the guards (and trips the fake device)
    e = _guard(m, force_all_rays=True)
    assert isinstance(e, AssertionError)


def test_shape_guards():
    m = _torso_model()
    for kw in ({"rays_o": torch.zeros(4, 2)}, {"rays_d": torch.zeros(5, 3)}, {"rays_o": torch.zeros(0, 3), "rays_d": torch.zeros(0, 3)},
               {"cond_feat": torch.zeros(63)}, {"ind_code": None}, {"ind_code": torch.zeros(3)}, {"max_steps": 0}, {"max_steps": 5000}):
        e = _guard(m, **kw)
        assert isinstance(e, ValueError), (kw, e)
    # a model without individual codes takes None
    m.individual_embedding_dim = 0
    e = _guard(m, ind_code=torch.zeros(4))
    assert isinstance(e, ValueError) and "ind_code" in str(e)
