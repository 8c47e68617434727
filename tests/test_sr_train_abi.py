"""gfpp_sr_forward_train / gfpp_sr_backward (gfpp.h section O) report bad arguments through the status code + gfpp_last_error()
before any CUDA call, so none of this needs a GPU."""
import ctypes

from genefaceplusplus_b200 import _capi

SR_MAGIC = 0x67667372      # what gfpp_sr_pack writes first ("gfsr")
P = ctypes.c_void_p


def _grad():
    g = _capi.SrGrad()
    g.conv_in_w = g.conv0_w = g.up_w = g.conv1_w = g.noise_strength = 4096
    for i in range(4):
        g.bias[i] = 4096
    for i in range(2):
        g.rgb_w[i] = g.rgb_b[i] = 4096
    return g


def _bwd(L, model, n_frames=1, in_res=256, saved_bytes=1 << 40, grad_out=P(4096), grad_in=P(4096), grad=None, ws_bytes=1 << 40):
    return L.gfpp_sr_backward(model, n_frames, in_res, P(4096), P(4096), saved_bytes, None, 0, grad_out, grad_in,
                              None if grad is None else ctypes.byref(grad), P(4096), ws_bytes, None)


def test_sr_backward_validates_before_any_cuda_call():
    L = _capi.lib()
    m = _capi.SrModel()
    m.opaque[0] = SR_MAGIC
    assert _bwd(L, ctypes.byref(m), grad_out=None) == -1 and b"null pointer" in L.gfpp_last_error()
    assert _bwd(L, ctypes.byref(m), grad_in=None) == -1 and b"neither" in L.gfpp_last_error()
    g = _grad()
    g.up_w = None
    assert _bwd(L, ctypes.byref(m), grad=g) == -1 and b"null gradient" in L.gfpp_last_error()
    for in_res in (0, 200, 2048):
        assert _bwd(L, ctypes.byref(m), in_res=in_res) == -4 and b"multiple of 128" in L.gfpp_last_error()
    assert _bwd(L, ctypes.byref(m), n_frames=0) == -4
    saved = L.gfpp_sr_train_workspace_bytes(2, 256)
    assert saved > L.gfpp_sr_workspace_bytes(2, 256)          # the training forward also keeps block1.conv1's activation
    assert _bwd(L, ctypes.byref(m), n_frames=2, saved_bytes=saved - 1) == -3 and b"saved" in L.gfpp_last_error()
    need = L.gfpp_sr_backward_workspace_bytes(2, 256)
    assert _bwd(L, ctypes.byref(m), n_frames=2, saved_bytes=saved, ws_bytes=need - 1) == -3
    assert b"workspace too small" in L.gfpp_last_error()
    # a handle gfpp_sr_pack never wrote is refused once the shapes pass
    assert _bwd(_capi.lib(), ctypes.byref(_capi.SrModel()), grad=_grad()) == -1 and b"gfpp_sr_pack" in L.gfpp_last_error()


def test_sr_forward_train_validates_before_any_cuda_call():
    L = _capi.lib()
    m = _capi.SrModel()
    m.opaque[0] = SR_MAGIC
    f = L.gfpp_sr_forward_train
    assert f(ctypes.byref(m), 1, 256, P(4096), None, 0, None, P(4096), 1 << 40, None) == -1
    assert f(ctypes.byref(m), 1, 200, P(4096), None, 0, P(4096), P(4096), 1 << 40, None) == -4
    need = L.gfpp_sr_train_workspace_bytes(1, 256)
    assert f(ctypes.byref(m), 1, 256, P(4096), None, 0, P(4096), P(4096), need - 1, None) == -3
    assert b"workspace too small" in L.gfpp_last_error()
