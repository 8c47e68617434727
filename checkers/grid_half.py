"""checkers/grid_half.py -- TEST INFRASTRUCTURE: ctypes wrappers over checkers/_build/libgridhalf.so, the C restatement of the
grid encoder on half tables (grid_half.c).  CPU torch tensors in and out; half tensors are accepted wherever the reference
passes half buffers and are widened to fp32 (exactly) before the call.

rnd=True is the half kernels' arithmetic (binary16 round-to-nearest-even at every at::Half rounding site); rnd=False evaluates
the same expressions in fp32 without 16-bit rounding.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "grid_half.c")
_LIB_PATH = os.path.join(_HERE, "_build", "libgridhalf.so")
_lib = None

P = ctypes.c_void_p
u32 = ctypes.c_uint32


def _compile(out):
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.run(["cc", "-O2", "-std=c11", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", out, "-lm"], check=True,
                   capture_output=True)


def build(force: bool = False) -> str:
    """Compile the checker into checkers/_build (cc only)."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        _compile(_LIB_PATH)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        path = _LIB_PATH
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(_SRC):
            try:
                build()
            except OSError:            # a read-only tree: build beside the process instead
                path = os.path.join(tempfile.mkdtemp(prefix="gridhalf_"), "libgridhalf.so")
                _compile(path)
        L = ctypes.CDLL(path)
        L.ghc_round_half.restype = ctypes.c_float
        L.ghc_round_half.argtypes = [ctypes.c_float]
        L.ghc_forward.argtypes = [P, P, P, u32, u32, u32, ctypes.c_float, u32, u32, ctypes.c_int, u32, P, ctypes.c_int, P, P]
        L.ghc_table_grad.argtypes = [P, P, P, u32, u32, u32, ctypes.c_float, u32, u32, ctypes.c_int, u32, P, ctypes.c_int, P, P, P]
        L.ghc_input_grad.argtypes = [P, P, u32, u32, u32, ctypes.c_int, P]
        _lib = L
    return _lib


def _f32(t):
    t = t.detach().cpu()
    assert t.dtype in (torch.float32, torch.float16), t.dtype
    return t.float().contiguous()


def _ptr(t):
    return P(t.data_ptr())


def _scales(scales):
    return None if scales is None else _f32(torch.as_tensor(scales, dtype=torch.float32))


def forward(inputs, emb, offsets, S, H, gridtype=1, align_corners=False, interp=0, dy_dx=False, rnd=True, scales=None):
    """outputs [L,B,2] and dy_dx [B,L,D,2] (or None) as fp32 tensors (binary16 values when rnd)."""
    x, e = _f32(inputs), _f32(emb)
    off = torch.as_tensor(offsets).to(torch.int32).contiguous()
    B, D = x.shape
    L = off.numel() - 1
    out = torch.empty(L, B, 2)
    dd = torch.empty(B, L, D, 2) if dy_dx else None
    sc = _scales(scales)
    rc = lib().ghc_forward(_ptr(x), _ptr(e), _ptr(off), B, D, L, float(S), H, gridtype, int(align_corners), interp,
                           None if sc is None else _ptr(sc), int(rnd), _ptr(out), None if dd is None else _ptr(dd))
    assert rc == 0
    return out, dd


def table_grad(grad, inputs, offsets, n_entries, S, H, gridtype=1, align_corners=False, interp=0, rnd=True, scales=None):
    """(float64 sum of the added terms [n,2], float64 sum of their magnitudes [n,2], adds per entry [n])."""
    g, x = _f32(grad), _f32(inputs)
    off = torch.as_tensor(offsets).to(torch.int32).contiguous()
    B, D = x.shape
    L = off.numel() - 1
    s = torch.zeros(n_entries, 2, dtype=torch.float64)
    a = torch.zeros(n_entries, 2, dtype=torch.float64)
    k = torch.zeros(n_entries, dtype=torch.int32)
    sc = _scales(scales)
    rc = lib().ghc_table_grad(_ptr(g), _ptr(x), _ptr(off), B, D, L, float(S), H, gridtype, int(align_corners), interp,
                              None if sc is None else _ptr(sc), int(rnd), _ptr(s), _ptr(a), _ptr(k))
    assert rc == 0
    return s, a, k


def input_grad(grad, dy_dx, rnd=True):
    """grad [L,B,2], dy_dx [B,L,D,2] -> grad_inputs [B,D]."""
    g, d = _f32(grad), _f32(dy_dx)
    B, L, D, _ = d.shape
    out = torch.empty(B, D)
    assert lib().ghc_input_grad(_ptr(g), _ptr(d), B, D, L, int(rnd), _ptr(out)) == 0
    return out


def round_half(v: float) -> float:
    return float(lib().ghc_round_half(ctypes.c_float(v)))


def ulp16(x):
    """binary16 ulp of |x| (elementwise, numpy or torch); 2^-24 below the normal range."""
    a = np.abs(np.asarray(x, dtype=np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.exp2(np.minimum(e, 15) - 10)
