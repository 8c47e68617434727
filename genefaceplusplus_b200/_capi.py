"""ctypes binding of libgfpp.so (the C-ABI declared in include/gfpp.h).

PyTorch is only plumbing here: device memory (`tensor.data_ptr()`), the current stream and
torch.distributed.  There is NO fallback: if the library is missing or a call fails, an exception is
raised (`GfppError`), never a silent CPU / eager path.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgfpp.so")
_lib = None

c_void_p = ctypes.c_void_p
c_u32 = ctypes.c_uint32
c_f = ctypes.c_float
c_int = ctypes.c_int
c_size_t = ctypes.c_size_t


class GfppError(RuntimeError):
    pass


class GfppNoCpuPath(GfppError, NotImplementedError):
    """A libgfpp entry point was called on a model that lives on the CPU: there is no CPU path."""


class GridDesc(ctypes.Structure):
    _fields_ = [("embeddings", c_void_p), ("offsets_host", c_void_p), ("input_dim", c_u32), ("num_levels", c_u32),
                ("base_resolution", c_u32), ("log2_per_level_scale", c_f), ("gridtype", c_u32), ("interp", c_u32),
                ("align_corners", c_int)]


class ModelDesc(ctypes.Structure):
    _fields_ = [("position_grid", GridDesc), ("ambient_grid", GridDesc),
                ("ambient_w", c_void_p * 3), ("sigma_w", c_void_p * 3), ("color_w", c_void_p * 2),
                ("individual_code", c_void_p), ("cond_dim", c_u32), ("ind_dim", c_u32),
                ("density_bitfield", c_void_p), ("aabb", c_f * 6), ("bound", c_f), ("min_near", c_f),
                ("cascade", c_u32), ("grid_size", c_u32), ("density_scale", c_f),
                ("has_torso", c_int), ("torso_grid", GridDesc),
                ("torso_deform_w", c_void_p * 3), ("torso_canon_w", c_void_p * 3), ("torso_code", c_void_p),
                ("density_grid_torso", c_void_p), ("density_thresh_torso", c_f), ("torso_shrink", c_f),
                ("torso_code_dim", c_u32), ("mlp_precision", c_u32)]


class Model(ctypes.Structure):
    _fields_ = [("opaque", ctypes.c_uint64 * 512)]


class Frames(ctypes.Structure):
    _fields_ = [("n_frames", c_u32), ("n_rays", c_u32), ("rays_o", c_void_p), ("rays_d", c_void_p),
                ("poses_c2w", c_void_p), ("fx", c_f), ("fy", c_f), ("cx", c_f), ("cy", c_f),
                ("img_h", c_u32), ("img_w", c_u32), ("cond_feat", c_void_p), ("torso_pose6", c_void_p),
                ("bg_coords", c_void_p), ("bg_color", c_void_p), ("dt_gamma", c_f), ("max_steps", c_u32),
                ("T_thresh", c_f), ("noises", c_void_p)]


class SrDesc(ctypes.Structure):
    _fields_ = [("conv_in_w", c_void_p), ("conv0_w", c_void_p), ("up_w", c_void_p), ("conv1_w", c_void_p),
                ("bias", c_void_p * 4), ("rgb_w", c_void_p * 2), ("rgb_b", c_void_p * 2)]


class SrModel(ctypes.Structure):
    _fields_ = [("opaque", ctypes.c_uint64 * 32)]


class TorsoSrDesc(ctypes.Structure):
    _fields_ = [("torso_grid", GridDesc), ("torso_deform_w", c_void_p * 3), ("torso_canon_w", c_void_p * 3), ("torso_code", c_void_p),
                ("torso_code_dim", c_u32), ("head_aware", c_int), ("ha_w", c_void_p * 3), ("ha_b", c_void_p * 3),
                ("density_grid_torso", c_void_p), ("grid_size", c_u32), ("density_thresh_torso", c_f), ("torso_shrink", c_f)]


class TorsoSrModel(ctypes.Structure):
    _fields_ = [("opaque", ctypes.c_uint64 * 128)]


class TorsoSrFrames(ctypes.Structure):
    _fields_ = [("n_frames", c_u32), ("n_rays", c_u32), ("image", c_void_p), ("weights_sum", c_void_p), ("lm68", c_void_p),
                ("bg_coords", c_void_p), ("bg_color", c_void_p)]


class Outputs(ctypes.Structure):
    _fields_ = [("rgb_map", c_void_p), ("depth_map", c_void_p), ("weights_sum", c_void_p),
                ("torso_alpha_map", c_void_p), ("torso_rgb_map", c_void_p), ("torso_deform", c_void_p),
                ("stats", c_void_p), ("rgb_u8", c_void_p), ("alpha_map", c_void_p), ("rgba_u8", c_void_p)]


EXPORTS = [
    "gfpp_last_error", "gfpp_version", "gfpp_check_device", "gfpp_near_far_from_aabb", "gfpp_march_rays",
    "gfpp_composite_rays", "gfpp_grid_encode_forward", "gfpp_sh_encode_forward", "gfpp_freq_encode_forward",
    "gfpp_model_packed_bytes", "gfpp_model_pack", "gfpp_render_workspace_bytes", "gfpp_render_frames",
    "gfpp_last_launch_count", "gfpp_profile_enable", "gfpp_profile_read", "gfpp_profile_phases", "gfpp_tc_selftest", "gfpp_debug_generate_rays",
    "gfpp_sr_packed_bytes", "gfpp_sr_pack", "gfpp_sr_workspace_bytes", "gfpp_sr_forward", "gfpp_sr_forward_video",
    "gfpp_torso_sr_packed_bytes", "gfpp_torso_sr_pack", "gfpp_torso_sr_workspace_bytes", "gfpp_torso_sr_composite",
    "gfpp_march_rays_train_scratch_bytes", "gfpp_march_rays_train", "gfpp_march_rays_train_backward", "gfpp_composite_rays_train_forward",
    "gfpp_composite_rays_train_backward", "gfpp_grid_encode_forward_dydx", "gfpp_grid_encode_backward", "gfpp_grad_total_variation",
    "gfpp_packbits", "gfpp_morton3D", "gfpp_morton3D_invert", "gfpp_morton3D_dilation", "gfpp_sph_from_ray",
    "gfpp_density_query", "gfpp_density_grid_workspace_bytes", "gfpp_density_grid_update", "gfpp_mark_untrained_grid",
    "gfpp_torso_grid_workspace_bytes", "gfpp_torso_query_workspace_bytes", "gfpp_torso_query", "gfpp_torso_grid_update", "gfpp_torso_sr_grid_update",
    "gfpp_model_set_torso_threshold", "gfpp_torso_sr_set_threshold",
    "gfpp_field_backward_workspace_bytes", "gfpp_field_forward", "gfpp_field_backward",
    "gfpp_field_tc_workspace_bytes", "gfpp_field_tc_forward", "gfpp_field_tc_backward",
    "gfpp_torso_field_workspace_bytes", "gfpp_torso_field_forward", "gfpp_torso_field_backward",
    "gfpp_torso_sr_field_workspace_bytes", "gfpp_torso_sr_field_forward", "gfpp_torso_sr_field_backward",
    "gfpp_frozen_head_workspace_bytes", "gfpp_frozen_head",
    "gfpp_grid_encode_forward_half", "gfpp_grid_encode_backward_half",
    "gfpp_torso_pass_workspace_bytes", "gfpp_torso_mask", "gfpp_torso_composite_forward", "gfpp_torso_composite_backward",
]


def lib():
    """Load libgfpp.so.  Fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GfppError(f"{LIB_PATH} not found: build it with `python -m genefaceplusplus_b200.build` "
                            "(there is no CPU or eager fallback)")
        L = ctypes.CDLL(LIB_PATH)
        L.gfpp_last_error.restype = ctypes.c_char_p
        L.gfpp_model_packed_bytes.restype = c_size_t
        L.gfpp_render_workspace_bytes.restype = c_size_t
        L.gfpp_model_packed_bytes.argtypes = [ctypes.POINTER(ModelDesc)]
        L.gfpp_model_pack.argtypes = [ctypes.POINTER(ModelDesc), c_void_p, c_size_t, ctypes.POINTER(Model), c_void_p]
        L.gfpp_render_workspace_bytes.argtypes = [c_u32, c_u32, c_u32]
        L.gfpp_render_frames.argtypes = [ctypes.POINTER(Model), ctypes.POINTER(Frames), ctypes.POINTER(Outputs), c_void_p,
                                         c_size_t, c_void_p]
        L.gfpp_near_far_from_aabb.argtypes = [c_void_p, c_void_p, c_void_p, c_u32, c_f, c_void_p, c_void_p, c_void_p]
        L.gfpp_march_rays.argtypes = [c_u32, c_u32, c_void_p, c_void_p, c_void_p, c_void_p, c_f, c_f, c_u32, c_u32, c_u32,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
        L.gfpp_composite_rays.argtypes = [c_u32, c_u32, c_f, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p]
        L.gfpp_grid_encode_forward.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_u32, c_u32, c_u32, c_u32, c_f, c_u32,
                                               c_u32, c_int, c_u32, c_void_p]
        L.gfpp_sh_encode_forward.argtypes = [c_void_p, c_void_p, c_u32, c_u32, c_u32, c_void_p]
        L.gfpp_freq_encode_forward.argtypes = [c_void_p, c_u32, c_u32, c_u32, c_u32, c_void_p, c_void_p]
        L.gfpp_profile_phases.argtypes = [c_void_p]
        L.gfpp_debug_generate_rays.argtypes = [c_void_p, c_u32, c_f, c_f, c_f, c_f, c_u32, c_u32, c_void_p, c_void_p, c_void_p]
        L.gfpp_tc_selftest.argtypes = [c_void_p, c_void_p, c_u32, c_u32, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.gfpp_sr_packed_bytes.restype = c_size_t
        L.gfpp_sr_packed_bytes.argtypes = []
        L.gfpp_sr_pack.argtypes = [ctypes.POINTER(SrDesc), c_void_p, c_size_t, ctypes.POINTER(SrModel), c_void_p]
        L.gfpp_sr_workspace_bytes.restype = c_size_t
        L.gfpp_sr_workspace_bytes.argtypes = [c_u32, c_u32]
        L.gfpp_sr_forward.argtypes = [ctypes.POINTER(SrModel), c_u32, c_u32, c_void_p, ctypes.POINTER(c_void_p * 4), c_u32, c_void_p,
                                      c_int, c_void_p, c_size_t, c_void_p]
        L.gfpp_sr_forward_video.argtypes = [ctypes.POINTER(SrModel), c_u32, c_u32, c_void_p, ctypes.POINTER(c_void_p * 4), c_u32,
                                            c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
        L.gfpp_torso_sr_packed_bytes.restype = c_size_t
        L.gfpp_torso_sr_packed_bytes.argtypes = []
        L.gfpp_torso_sr_pack.argtypes = [ctypes.POINTER(TorsoSrDesc), c_void_p, c_size_t, ctypes.POINTER(TorsoSrModel), c_void_p]
        L.gfpp_torso_sr_workspace_bytes.restype = c_size_t
        L.gfpp_torso_sr_workspace_bytes.argtypes = [c_u32]
        L.gfpp_torso_sr_composite.argtypes = [ctypes.POINTER(TorsoSrModel), ctypes.POINTER(TorsoSrFrames), c_void_p, c_void_p, c_void_p,
                                              c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
        P = c_void_p
        L.gfpp_march_rays_train_scratch_bytes.restype = c_size_t
        L.gfpp_march_rays_train_scratch_bytes.argtypes = [c_u32]
        L.gfpp_march_rays_train.argtypes = [P, P, P, c_f, c_f, c_u32, c_u32, c_u32, c_u32, c_u32, P, P, P, P, P, P, P, P, P, c_size_t, P]
        L.gfpp_march_rays_train_backward.argtypes = [P, P, P, P, c_u32, c_u32, P, P, P]
        L.gfpp_composite_rays_train_forward.argtypes = [P, P, P, P, P, c_u32, c_u32, c_f, P, P, P, P, P]
        L.gfpp_composite_rays_train_backward.argtypes = [P, P, P, P, P, P, P, P, P, P, P, c_u32, c_u32, c_f, P, P, P, P]
        L.gfpp_grid_encode_forward_dydx.argtypes = [P, P, P, P, c_u32, c_u32, c_u32, c_u32, c_f, c_u32, P, c_u32, c_int, c_u32, P]
        L.gfpp_grid_encode_backward.argtypes = [P, P, P, P, P, c_u32, c_u32, c_u32, c_u32, c_f, c_u32, P, P, c_u32, c_int, c_u32, P]
        L.gfpp_grid_encode_forward_half.argtypes = [P, P, P, P, c_u32, c_u32, c_u32, c_u32, c_f, c_u32, P, c_u32, c_int, c_u32, P]
        L.gfpp_grid_encode_backward_half.argtypes = L.gfpp_grid_encode_backward.argtypes
        L.gfpp_grad_total_variation.argtypes = [P, P, P, P, c_f, c_u32, c_u32, c_u32, c_u32, c_f, c_u32, c_u32, c_int, P]
        L.gfpp_packbits.argtypes = [P, c_u32, c_f, P, P]
        L.gfpp_morton3D.argtypes = [P, c_u32, P, P]
        L.gfpp_morton3D_invert.argtypes = [P, c_u32, P, P]
        L.gfpp_morton3D_dilation.argtypes = [P, c_u32, c_u32, P, P]
        L.gfpp_sph_from_ray.argtypes = [P, P, c_f, c_u32, P, P]
        c_d = ctypes.c_double
        L.gfpp_density_query.argtypes = [ctypes.POINTER(Model), P, c_u32, P, P, P, P]
        L.gfpp_density_grid_workspace_bytes.restype = c_size_t
        L.gfpp_density_grid_workspace_bytes.argtypes = [c_u32, c_u32]
        L.gfpp_density_grid_update.argtypes = [ctypes.POINTER(Model), P, P, c_f, c_f, P, P, P, P, c_size_t, P]
        L.gfpp_mark_untrained_grid.argtypes = [P, c_u32, c_d, c_d, c_d, c_d, c_d, c_u32, c_u32, P, P]
        L.gfpp_torso_grid_workspace_bytes.restype = c_size_t
        L.gfpp_torso_grid_workspace_bytes.argtypes = [c_u32]
        L.gfpp_torso_query_workspace_bytes.restype = c_size_t
        L.gfpp_torso_query_workspace_bytes.argtypes = []
        L.gfpp_torso_query.argtypes = [ctypes.POINTER(Model), P, c_u32, P, P, P, P, P, P, c_size_t, P]
        L.gfpp_torso_grid_update.argtypes = [ctypes.POINTER(Model), P, P, P, c_f, P, P, P, P, c_size_t, P]
        L.gfpp_torso_sr_grid_update.argtypes = [ctypes.POINTER(TorsoSrModel), P, P, P, c_f, P, P, P, P, c_size_t, P]
        L.gfpp_model_set_torso_threshold.argtypes = [ctypes.POINTER(Model), c_f]
        L.gfpp_torso_sr_set_threshold.argtypes = [ctypes.POINTER(TorsoSrModel), c_f]
        L.gfpp_field_backward_workspace_bytes.restype = c_size_t
        L.gfpp_field_backward_workspace_bytes.argtypes = [c_u32]
        L.gfpp_field_forward.argtypes = [ctypes.POINTER(ModelDesc), P, P, c_u32, P, P, P, P, P, c_size_t, P]
        L.gfpp_field_backward.argtypes = [ctypes.POINTER(ModelDesc), P, P, c_u32, P, P, P, P, ctypes.POINTER(P * 8), P, P, P, P, P, c_size_t, P]
        L.gfpp_field_tc_workspace_bytes.restype = c_size_t
        L.gfpp_field_tc_workspace_bytes.argtypes = [c_u32]
        L.gfpp_field_tc_forward.argtypes = L.gfpp_field_forward.argtypes
        L.gfpp_field_tc_backward.argtypes = L.gfpp_field_backward.argtypes
        L.gfpp_frozen_head_workspace_bytes.restype = c_size_t
        L.gfpp_frozen_head_workspace_bytes.argtypes = [c_u32, c_u32]
        L.gfpp_frozen_head.argtypes = [ctypes.POINTER(Model), P, P, c_u32, ctypes.POINTER(c_f), P, P, P, c_f,
                                       c_u32, c_f, P, P, P, c_size_t, P]
        L.gfpp_torso_field_workspace_bytes.restype = c_size_t
        L.gfpp_torso_field_workspace_bytes.argtypes = [c_u32]
        L.gfpp_torso_field_forward.argtypes = [ctypes.POINTER(ModelDesc), P, c_u32, P, P, P, P, P, P, c_size_t, P]
        L.gfpp_torso_field_backward.argtypes = [ctypes.POINTER(ModelDesc), P, c_u32, P, P, P, P, P, ctypes.POINTER(P * 3),
                                                ctypes.POINTER(P * 3), P, P, P, c_size_t, P]
        L.gfpp_torso_sr_field_workspace_bytes.restype = c_size_t
        L.gfpp_torso_sr_field_workspace_bytes.argtypes = [c_u32]
        L.gfpp_torso_sr_field_forward.argtypes = [ctypes.POINTER(TorsoSrDesc), P, c_u32, P, P, P, P, P, P, P, P, c_size_t, P]
        L.gfpp_torso_sr_field_backward.argtypes = [ctypes.POINTER(TorsoSrDesc), P, c_u32, P, P, P, P, P, P, P, ctypes.POINTER(P * 3),
                                                   ctypes.POINTER(P * 3), ctypes.POINTER(P * 3), ctypes.POINTER(P * 3), P, P, P, c_size_t, P]
        L.gfpp_torso_pass_workspace_bytes.restype = c_size_t
        L.gfpp_torso_pass_workspace_bytes.argtypes = [c_u32]
        L.gfpp_torso_mask.argtypes = [P, c_u32, c_f, P, c_u32, P, P, P, P, P, P, P, P, P, c_size_t, P]
        L.gfpp_torso_composite_forward.argtypes = [P, c_u32, c_u32, P, P, P, P, P, c_u32, P, P, P, P]
        L.gfpp_torso_composite_backward.argtypes = [P, c_u32, c_u32, P, P, P, P, P, c_u32, P, P, P, P, P, P]
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        raise GfppError(f"{what} failed ({rc}): {lib().gfpp_last_error().decode()}")


def stream_ptr(device=None):
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t, dtype=None):
    """Device pointer of a contiguous CUDA tensor (or None)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise GfppError("expected a CUDA tensor (libgfpp has no CPU path)")
    if not t.is_contiguous():
        raise GfppError("expected a contiguous tensor")
    if dtype is not None and t.dtype != dtype:
        raise GfppError(f"expected dtype {dtype}, got {t.dtype}")
    return c_void_p(t.data_ptr())
