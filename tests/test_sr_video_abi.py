"""gfpp_sr_forward_video (gfpp.h section C): the SR head's video-frame entry point reports bad arguments through the status code +
gfpp_last_error() before any CUDA call, so none of this needs a GPU."""
import ctypes

from genefaceplusplus_b200 import _capi

SR_MAGIC = 0x67667372      # what gfpp_sr_pack writes first ("gfsr")
P = ctypes.c_void_p


def _call(L, model, n_frames=1, in_res=256, rgb=P(4096), out=P(4096), out_u8=P(4096), ws=P(4096), ws_bytes=1 << 40):
    return L.gfpp_sr_forward_video(model, n_frames, in_res, rgb, None, 0, out, out_u8, ws, ws_bytes, None)


def test_sr_forward_video_validates_before_any_cuda_call():
    L = _capi.lib()
    m = _capi.SrModel()
    assert L.gfpp_sr_forward_video(None, 1, 256, P(4096), None, 0, P(4096), P(4096), P(4096), 1 << 30, None) == -1
    assert b"sr_forward_video: null pointer" in L.gfpp_last_error()
    assert _call(L, ctypes.byref(m), rgb=None) == -1 and b"null" in L.gfpp_last_error()
    assert _call(L, ctypes.byref(m), ws=None) == -1 and b"null" in L.gfpp_last_error()
    assert _call(L, ctypes.byref(m), out=None, out_u8=None) == -1 and b"null" in L.gfpp_last_error()     # nothing to write
    assert _call(L, ctypes.byref(m), out_u8=P(4097)) == -1 and b"4-byte aligned" in L.gfpp_last_error()
    assert _call(L, ctypes.byref(m)) == -1 and b"gfpp_sr_pack" in L.gfpp_last_error()                    # handle never packed
    m.opaque[0] = SR_MAGIC
    for in_res in (0, 200, 2048):
        assert _call(L, ctypes.byref(m), in_res=in_res) == -4 and b"multiple of 128" in L.gfpp_last_error()
    assert _call(L, ctypes.byref(m), n_frames=0) == -4
    assert _call(L, ctypes.byref(m), n_frames=20000) == -4 and b"too many frames" in L.gfpp_last_error()
    need = L.gfpp_sr_workspace_bytes(2, 256)
    assert _call(L, ctypes.byref(m), n_frames=2, ws_bytes=need - 1) == -3 and b"workspace too small" in L.gfpp_last_error()
    # either output alone passes the argument checks (the workspace check is the last one before the launches)
    assert _call(L, ctypes.byref(m), out=None, ws_bytes=need - 1, n_frames=2) == -3
    assert _call(L, ctypes.byref(m), out_u8=None, ws_bytes=need - 1, n_frames=2) == -3


def test_sr_forward_keeps_its_messages_and_requires_out():
    L = _capi.lib()
    m = _capi.SrModel()
    m.opaque[0] = SR_MAGIC
    assert L.gfpp_sr_forward(ctypes.byref(m), 1, 256, P(4096), None, 0, None, 1, P(4096), 1 << 40, None) == -1
    assert b"sr_forward: null pointer" in L.gfpp_last_error()
    assert L.gfpp_sr_forward(ctypes.byref(m), 1, 200, P(4096), None, 0, P(4096), 1, P(4096), 1 << 40, None) == -4
    assert L.gfpp_last_error().startswith(b"sr_forward: in_res")
