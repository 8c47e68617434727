"""oracle/ref_train_shim.py -- TEST INFRASTRUCTURE: the opt-in training half of oracle/ref_shim.py.

install_training(ops), called after ref_shim.install(ops), lets the reference's training branch of NeRFRenderer.render and its
backward run on the CPU with the C restatement of its native ops (oracle/native_ops.c through oracle/ops.py):
  * `_raymarching_face.composite_rays_train_forward / _backward` (raymarching.h:16-17) -> orc_composite_rays_train_*; the reference's
    own autograd wrapper (raymarching.py:276-341) runs unchanged on top;
  * `_gridencoder.grid_encode_forward` with dy_dx and `grid_encode_backward` (gridencoder.h:12-13) -> orc_grid_encode_*; grid.py's
    autograd Function runs unchanged on top;
  * the wrapper `march_rays_train` (raymarching.py:184-270), which forces .cuda() and calls torch.cuda.empty_cache(), is replaced by
    its restatement on the CPU (same M / mean_count / align / noise logic; point offsets in ray order, the checker's layout).
ref_shim.install() itself is unchanged: the inference goldens never see these substitutions.
"""
import ctypes
import sys

import torch

u32 = ctypes.c_uint32


def install_training(ops):
    L = ops.lib()
    rmf = sys.modules["_raymarching_face"]

    def composite_rays_train_forward(sigmas, rgbs, ambient, deltas, rays, M, N, T_thresh, weights_sum, ambient_sum, depth, image):
        L.orc_composite_rays_train_forward(ops._f(sigmas), ops._f(rgbs), ops._f(ambient), ops._f(deltas), ops._i(rays), u32(M), u32(N),
                                           ctypes.c_float(T_thresh), ops._f(weights_sum), ops._f(ambient_sum), ops._f(depth), ops._f(image))

    def composite_rays_train_backward(g_ws, g_asum, g_image, sigmas, rgbs, ambient, deltas, rays, ws, asum, image, M, N, T_thresh, g_sigmas,
                                      g_rgbs, g_ambient):
        L.orc_composite_rays_train_backward(ops._f(g_ws), ops._f(g_asum), ops._f(g_image), ops._f(sigmas), ops._f(rgbs), ops._f(ambient),
                                            ops._f(deltas), ops._i(rays), ops._f(ws), ops._f(asum), ops._f(image), u32(M), u32(N),
                                            ctypes.c_float(T_thresh), ops._f(g_sigmas), ops._f(g_rgbs), ops._f(g_ambient))

    rmf.composite_rays_train_forward = composite_rays_train_forward
    rmf.composite_rays_train_backward = composite_rays_train_backward

    gmod = sys.modules["_gridencoder"]

    def grid_encode_forward(inputs, embeddings, offsets, outputs, B, D, C, Lv, S, H, dy_dx, gridtype, align_corners, interp):
        ops.grid_encode_forward_raw(inputs, embeddings, offsets, outputs, B, D, C, Lv, float(S), H, gridtype, align_corners, interp)
        if dy_dx is not None:
            rc = L.orc_grid_encode_dydx(ops._f(inputs), ops._f(embeddings), ops._i(offsets), ops._f(dy_dx), u32(B), u32(D), u32(C), u32(Lv),
                                        ctypes.c_float(float(S)), u32(H), u32(gridtype), ctypes.c_int(int(align_corners)), u32(interp))
            assert rc == 0

    def grid_encode_backward(grad, inputs, embeddings, offsets, grad_embeddings, B, D, C, Lv, S, H, dy_dx, grad_inputs, gridtype, align_corners,
                             interp):
        rc = L.orc_grid_encode_backward(ops._f(grad), ops._f(inputs), ops._i(offsets), ops._f(grad_embeddings), u32(B), u32(D), u32(C), u32(Lv),
                                        ctypes.c_float(float(S)), u32(H), ops._f(dy_dx) if dy_dx is not None else None,
                                        ops._f(grad_inputs) if grad_inputs is not None else None, u32(gridtype),
                                        ctypes.c_int(int(align_corners)), u32(interp))
        assert rc == 0

    gmod.grid_encode_forward = grid_encode_forward
    gmod.grid_encode_backward = grid_encode_backward

    def march_rays_train(rays_o, rays_d, bound, density_bitfield, C, H, nears, fars, step_counter=None, mean_count=-1, perturb=False, align=-1,
                         force_all_rays=False, dt_gamma=0, max_steps=1024):
        rays_o = rays_o.float().contiguous().view(-1, 3)
        rays_d = rays_d.float().contiguous().view(-1, 3)
        N = rays_o.shape[0]
        M = N * max_steps
        if not force_all_rays and mean_count > 0:
            if align > 0:
                mean_count += align - mean_count % align
            M = mean_count
        if step_counter is None:
            step_counter = torch.zeros(2, dtype=torch.int32)
        noises = torch.rand(N) if perturb else torch.zeros(N)
        xyzs, dirs, deltas, rays, _ = ops.march_rays_train(rays_o, rays_d, bound, density_bitfield.contiguous(), C, H, nears.float().contiguous(),
                                                           fars.float().contiguous(), M=M, noises=noises, dt_gamma=dt_gamma, max_steps=max_steps,
                                                           counter=step_counter)
        if force_all_rays or mean_count <= 0:
            m = int(step_counter[0].item())
            if align > 0:
                m += align - m % align
            xyzs, dirs, deltas = xyzs[:m], dirs[:m], deltas[:m]
        return xyzs, dirs, deltas, rays

    import modules.radnerfs.raymarching as rm  # noqa: E402
    import modules.radnerfs.raymarching.raymarching as rm_inner  # noqa: E402
    for target in (rm, rm_inner):
        target.march_rays_train = march_rays_train
