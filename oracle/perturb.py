"""oracle/perturb.py -- TEST INFRASTRUCTURE: the reference's perturb=True in the inference branch of render().

Follows (paths relative to the reference tree):
  march_rays wrapper        modules/radnerfs/raymarching/raymarching.py:376-392  (noises = torch.rand(n_alive) when perturb)
  march_rays kernel         modules/radnerfs/raymarching/src/raymarching.cu:873  (t += clamp(t*dt_gamma, dt_min, dt_max) * noise)
  render loop               modules/radnerfs/renderer.py:354-384, radnerf_torso.py:138-151, radnerf_torso_sr.py:166-181
                            (march_rays(..., perturb if step == 0 else False, ...))

`march_rays` restates the wrapper with its perturb branch on the C kernel, which already takes `noises`; with perturb=False it
is oracle.ops.march_rays.  `render` runs OracleModel.render (oracle/render.py, whose loop keeps the reference's round
structure) with the step-0 rule: the first march_rays call of the render gets the noise vector, every later one zeros.  An
explicit `noises` [N] lets the oracle and the GPU renderer share one draw; otherwise it is drawn as the reference does.
"""
import ctypes

import torch

from . import ops


def march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, density_bitfield, C, H, near, far,
               align=-1, perturb=False, dt_gamma=0, max_steps=1024, noises=None):
    """raymarching.py:376-392.  noises: optional explicit [n_alive] vector used in place of the draw (perturb must be truthy)."""
    if not perturb:
        assert noises is None
        return ops.march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, density_bitfield, C, H, near, far,
                              align, False, dt_gamma, max_steps)
    rays_o = rays_o.float().contiguous().view(-1, 3)
    rays_d = rays_d.float().contiguous().view(-1, 3)
    M = n_alive * n_step
    if align > 0:
        M += align - (M % align)
    xyzs = torch.zeros(M, 3, dtype=torch.float32)
    dirs = torch.zeros(M, 3, dtype=torch.float32)
    deltas = torch.zeros(M, 2, dtype=torch.float32)
    if noises is None:
        noises = torch.rand(n_alive, dtype=rays_o.dtype, device=rays_o.device)
    noises = noises.float().contiguous().cpu()
    assert noises.numel() == n_alive, (noises.numel(), n_alive)
    ops.lib().orc_march_rays(ops.u32(n_alive), ops.u32(n_step), ops._i(rays_alive), ops._f(rays_t), ops._f(rays_o), ops._f(rays_d),
                             ctypes.c_float(bound), ctypes.c_float(dt_gamma), ops.u32(max_steps), ops.u32(C), ops.u32(H),
                             ops._b(density_bitfield), ops._f(near), ops._f(far), ops._f(xyzs), ops._f(dirs), ops._f(deltas),
                             ops._f(noises))
    return xyzs, dirs, deltas


class _StepZeroJitter:
    """The native-op backend of OracleModel with the reference's step-0 rule: the first march_rays call is perturbed with
    `noises`, every later call is not (raymarching.py:388-392 then draws nothing and passes zeros)."""

    def __init__(self, base, noises):
        self._base, self._noises = base, noises
        self.used = None

    def __getattr__(self, name):
        return getattr(self._base, name)

    def march_rays(self, n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, density_bitfield, C, H, near, far,
                   align=-1, perturb=False, dt_gamma=0, max_steps=1024):
        assert not perturb
        if self.used is None:
            # the first round: all N rays alive (renderer.py:349-351), one draw of n_alive values unless given
            noises = self._noises if self._noises is not None else torch.rand(n_alive, dtype=torch.float32)
            self.used = noises.float().reshape(-1).clone()
            return march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, density_bitfield, C, H, near, far,
                              align, True, dt_gamma, max_steps, noises=self.used)
        return self._base.march_rays(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, density_bitfield, C, H,
                                     near, far, align, False, dt_gamma, max_steps)


def render(orc, *args, perturb=True, noises=None, **kwargs):
    """OracleModel.render(*args, perturb=perturb, **kwargs) with the reference's perturb semantics.  noises: optional [N]
    (drawn with torch.rand(N) at the first round otherwise, after every host op that precedes it and before the SR head's noise
    planes).  The result gets `noises`: the vector used (None with perturb=False)."""
    if not perturb:
        assert noises is None
        res = orc.render(*args, perturb=False, **kwargs)
        res["noises"] = None
        return res
    base = orc.ops
    jit = _StepZeroJitter(base, noises)
    orc.ops = jit
    try:
        res = orc.render(*args, perturb=False, **kwargs)
    finally:
        orc.ops = base
    res["noises"] = jit.used
    return res
