"""Workspace of the pass-1 sample lists (k_march_list, DESIGN §5), without a GPU: every ray of a render call has a 64-byte list entry
(HIT_TS = 16 words) beside its 64-byte hit record, in the workspace size gfpp_render_workspace_bytes reports."""
import pytest

from genefaceplusplus_b200 import _capi

N = 1 << 16   # a multiple of the layouts' 256-byte alignment for every per-ray array


@pytest.fixture(scope="module")
def L():
    from genefaceplusplus_b200 import build
    build.build()
    return _capi.lib()


@pytest.mark.parametrize("F", [1, 3, 50])
def test_render_workspace_per_ray(L, F):
    # image 12 + rays_t 4 + weights_sum 4 + depth 4 + survivors 4 + hit record 64 + sample list 64 bytes per ray
    grow = L.gfpp_render_workspace_bytes(F, 2 * N, 16) - L.gfpp_render_workspace_bytes(F, N, 16)
    assert grow == F * N * (12 + 4 + 4 + 4 + 4 + 64 + 64)

