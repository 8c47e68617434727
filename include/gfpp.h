/*
 * gfpp.h -- C-ABI of libgfpp.so: the H100 (sm_90a) render hot path of GeneFace++.
 *
 * Drop-in boundary (SURVEY.md section 8(b)).  Plain pointers and sizes only; no torch types.
 * All pointers are DEVICE pointers unless the name ends in _host.  Every call is
 * stream-ordered on `stream` (a cudaStream_t passed as void*), never synchronises the
 * device, never allocates device memory (callers provide packed-model and workspace
 * buffers whose sizes they query first) and never throws: the return value is 0 on success
 * or a negative gfpp_status; gfpp_last_error() returns a thread-local message.
 *
 * Two levels are exported.
 *
 *  (A) per-op entry points that mirror, argument for argument, the pybind functions of the
 *      reference's four CUDA extensions, so the reference's own Python wrappers can bind them
 *      (INTEGRATION.md shows the stub):
 *        gfpp_near_far_from_aabb   <- modules/radnerfs/raymarching/src/raymarching.h:7  (raymarching.cu:148-156)
 *        gfpp_march_rays           <- raymarching.h:19 (raymarching.cu:932-939)
 *        gfpp_composite_rays       <- raymarching.h:20 (raymarching.cu:1032-1037)
 *        gfpp_grid_encode_forward  <- modules/radnerfs/encoders/gridencoder/src/gridencoder.h:12 (gridencoder.cu:446-471)
 *        gfpp_sh_encode_forward    <- modules/radnerfs/encoders/shencoder/src/shencoder.h:9 (shencoder.cu:400)
 *        gfpp_freq_encode_forward  <- modules/radnerfs/encoders/freqencoder/src/freqencoder.h:7 (freqencoder.cu:97-110)
 *
 *  (B) the fused frame renderer that replaces the whole host-driven loop of
 *      NeRFRenderer.render / RADNeRFTorso.render (modules/radnerfs/renderer.py:340-399,
 *      modules/radnerfs/radnerf_torso.py:129-197) for one or many frames per call:
 *        gfpp_model_packed_bytes / gfpp_model_pack / gfpp_render_workspace_bytes / gfpp_render_frames
 *
 *  (C) the SR checkpoints' extra stages (SURVEY.md 8(f) rank 3): gfpp_sr_* (256 -> 512 super-resolution head) and
 *      gfpp_torso_sr_* (the torso field of radnerf_torso_sr.py), declared at the end of this file.
 *
 *  (D) the training-side native ops (SURVEY.md 8(f) rank 4), mirroring the reference's pybind functions like (A).
 *
 *  (E) occupancy-grid maintenance of the head models: density query, grid refresh, mark_untrained_grid.
 *
 *  (F) the torso models' occupancy grid: torso field query and density_grid_torso refresh, threshold setters.
 *
 *  (G) the trainable head field: RADNeRF.forward and its backward at explicit points, fp32.
 *
 *  (H) the trainable torso field: RADNeRFTorso.forward_torso and its backward at explicit points, fp32.
 *
 *  (I) the trainable torso-SR field: RADNeRFTorsowithSR.forward_torso and its backward at explicit points, fp32.
 *
 *  (J) the trainable head field of (G) on tensor cores: fp16 operands, fp32 accumulation, fp32 parameters and gradients.
 *
 *  (K) the frozen head of the torso training steps.
 *
 *  (L) the grid encoder ops of (A) and (D) on half tables, as the reference runs them under autocast.
 *
 *  (M) the torso pass of the torso training steps: mask, compaction and composite between (K) and the fields of (H) / (I).
 *
 *  (O) the gradients of the SR head of (C): a training forward that keeps its activations and the backward on TF32 tensor cores.
 */
#ifndef GFPP_H_
#define GFPP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GFPP_API __attribute__((visibility("default")))

typedef enum {
    GFPP_OK = 0,
    GFPP_ERR_INVALID = -1,     /* bad argument (null pointer, unsupported C/D/degree, size mismatch) */
    GFPP_ERR_CUDA = -2,        /* a CUDA runtime call failed; see gfpp_last_error() */
    GFPP_ERR_WORKSPACE = -3,   /* caller-provided buffer too small */
    GFPP_ERR_UNSUPPORTED = -4  /* configuration outside what the kernels were built for */
} gfpp_status;

GFPP_API const char *gfpp_last_error(void);
GFPP_API int gfpp_version(void);
/* device check: returns GFPP_OK iff the current device is compute capability 10.x */
GFPP_API int gfpp_check_device(void);

/* ------------------------------------------------------------------ (A) per-op mirror */

/* nears/fars [N] <- slab test of rays [N,3] against aabb[6]; miss => both FLT_MAX; near >= min_near */
GFPP_API int gfpp_near_far_from_aabb(const float *rays_o, const float *rays_d, const float *aabb, uint32_t N,
                                     float min_near, float *nears, float *fars, void *stream);

/* one round of inference marching: for each of n_alive rays emit up to n_step occupied samples.
 * xyzs/dirs [M,3] and deltas [M,2] must be zero-initialised by the caller (as the reference wrapper does). */
GFPP_API int gfpp_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t *rays_alive, const float *rays_t,
                             const float *rays_o, const float *rays_d, float bound, float dt_gamma,
                             uint32_t max_steps, uint32_t C, uint32_t H, const uint8_t *grid, const float *nears,
                             const float *fars, float *xyzs, float *dirs, float *deltas, const float *noises,
                             void *stream);

/* front-to-back compositing of one round, in place; kills rays by writing -1 into rays_alive */
GFPP_API int gfpp_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t *rays_alive,
                                 float *rays_t, const float *sigmas, const float *rgbs, const float *deltas,
                                 float *weights_sum, float *depth, float *image, void *stream);

/* multi-resolution grid encode, forward only.  inputs [B,D] in [0,1]; embeddings [sum,C] fp32;
 * offsets_host [L+1] (HOST pointer: the level layout is tiny and static); outputs [L,B,C] (L-major,
 * exactly what the reference kernel writes).  D in {2,3}, C == 2 (the only shapes on the path). */
GFPP_API int gfpp_grid_encode_forward(const float *inputs, const float *embeddings, const int32_t *offsets_host,
                                      float *outputs, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S,
                                      uint32_t H, uint32_t gridtype, int align_corners, uint32_t interp, void *stream);

/* real spherical harmonics, degree (called C in the reference) 1..4: outputs [B, degree^2] */
GFPP_API int gfpp_sh_encode_forward(const float *inputs, float *outputs, uint32_t B, uint32_t D, uint32_t degree,
                                    void *stream);

/* [x, sin(2^f x), sin(2^f x + pi/2)]_f : outputs [B, C], C = D + 2*D*deg */
GFPP_API int gfpp_freq_encode_forward(const float *inputs, uint32_t B, uint32_t D, uint32_t deg, uint32_t C,
                                      float *outputs, void *stream);

/* ------------------------------------------------------------------ (B) fused renderer */

/* One multi-resolution grid in the reference layout (GridEncoder, grid.py:98-136). */
typedef struct {
    const float *embeddings;      /* device [n_entries, 2] fp32 */
    const int32_t *offsets_host;  /* host   [num_levels+1] */
    uint32_t input_dim;           /* 2 or 3 */
    uint32_t num_levels;          /* <= 16 */
    uint32_t base_resolution;     /* H (16) */
    float log2_per_level_scale;   /* S, as float32(log2(per_level_scale)) */
    uint32_t gridtype;            /* 0 hash, 1 tiled */
    uint32_t interp;              /* 0 linear, 1 smoothstep */
    int align_corners;
} gfpp_grid_desc;

/* Weights in the reference's nn.Linear layout [out, in], fp32, device pointers (state_dict tensors). */
typedef struct {
    /* head field (modules/radnerfs/radnerf.py:56-86) */
    gfpp_grid_desc position_grid;       /* 3-D */
    gfpp_grid_desc ambient_grid;        /* ambient_coord_dim-D (3 for the May configs) */
    const float *ambient_w[3];          /* (128,96) (128,128) (3,128) */
    const float *sigma_w[3];            /* (128,64) (128,128) (129,128) */
    const float *color_w[2];            /* (128,148) (3,128) */
    const float *individual_code;       /* [ind_dim] = individual_embeddings[0]; may be NULL if ind_dim == 0 */
    uint32_t cond_dim;                  /* 64 */
    uint32_t ind_dim;                   /* 4 */
    /* occupancy + marching (modules/radnerfs/renderer.py:67-102) */
    const uint8_t *density_bitfield;    /* [cascade * grid_size^3 / 8], Morton order */
    float aabb[6];
    float bound;
    float min_near;
    uint32_t cascade;
    uint32_t grid_size;
    float density_scale;
    /* torso field (modules/radnerfs/radnerf_torso.py:17-49); has_torso == 0 for head-only RADNeRF */
    int has_torso;
    gfpp_grid_desc torso_grid;          /* 2-D */
    const float *torso_deform_w[3];     /* (64,104) (64,64) (2,64) */
    const float *torso_canon_w[3];      /* (32,136) (32,32) (4,32) */
    const float *torso_code;            /* [8] = torso_individual_codes[0] */
    const float *density_grid_torso;    /* [grid_size^2] */
    float density_thresh_torso;         /* min(density_thresh_torso, mean_density_torso) as the reference evaluates it */
    float torso_shrink;
    uint32_t torso_code_dim;            /* 8 */
    /* arithmetic of the head MLP GEMMs: 0 = fp32 FFMA (CUDA cores), 1 = fp16 operands on wgmma tensor cores with
     * fp32 accumulation (what the reference runs under autocast), 2 = bf16 hi/lo split x3 on wgmma (~fp32 accuracy),
     * 3 = bf16 x1, 4 = "robust": fp16 on wgmma with the hi/lo split (3 MMAs per k-step, ~22 mantissa bits) on the ambient
     * net only and a 16-bit fixed-point position table -- the two roundings the field amplifies; holds 1e-3 max-abs on
     * well-conditioned (trained-like) scenes where plain fp16 does not.  Modes 1 and 4 run the row-owner kernel
     * (head_v2_kernel.cu).  Everything else (marching, compositing, torso) is fp32 in every mode. */
    uint32_t mlp_precision;
} gfpp_model_desc;

/* Host-side model handle: plain data, caller-allocated (stack, heap, numpy buffer ...), filled by
 * gfpp_model_pack().  It holds level tables, launch constants and device pointers into `packed` and into
 * the borrowed tables; copying it is fine, it owns nothing. */
typedef struct gfpp_model {
    uint64_t opaque[512];
} gfpp_model;

/* bytes of the device buffer gfpp_model_pack() fills (repacked/transposed weights, occupancy bounds) */
GFPP_API size_t gfpp_model_packed_bytes(const gfpp_model_desc *desc);
/* Repack on `stream` into `packed` (device, >= gfpp_model_packed_bytes) and fill *model.  Weights are copied
 * (k-major, layer chunks in streaming order); the desc's grid tables, bitfield and density_grid_torso are
 * BORROWED and must stay alive while the model is used.  Unsupported layer shapes => GFPP_ERR_UNSUPPORTED
 * (the kernels are built for the May architecture: hidden 128, cond 64, geo 128, 16 levels x 2 features). */
GFPP_API int gfpp_model_pack(const gfpp_model_desc *desc, void *packed, size_t packed_bytes, gfpp_model *model,
                             void *stream);

typedef struct {
    uint32_t n_frames;            /* F */
    uint32_t n_rays;              /* N = H*W rays per frame */
    /* rays: either supplied (parity on identical rays) ... */
    const float *rays_o;          /* [F,N,3] or NULL */
    const float *rays_d;          /* [F,N,3] or NULL */
    /* ... or generated in-kernel from the camera (get_rays, modules/radnerfs/utils.py:283-364) */
    const float *poses_c2w;       /* [F,4,4] row-major; used when rays_o == NULL */
    float fx, fy, cx, cy;
    uint32_t img_h, img_w;
    const float *cond_feat;       /* [F,cond_dim] output of cal_cond_feat (radnerf.py:88-106) */
    const float *torso_pose6;     /* [F,6] euler+trans from convert_poses; NULL if no torso */
    const float *bg_coords;       /* [N,2] (shared by all frames); NULL if no torso */
    const float *bg_color;        /* [N,3] shared by all frames, or NULL => 1.0 (renderer.py:387-388) */
    float dt_gamma;
    uint32_t max_steps;
    float T_thresh;
    const float *noises;          /* [F,N] in [0,1), or NULL = no jitter (renderer.py:370, raymarching.py:388-392) */
} gfpp_frames;

typedef struct {
    float *rgb_map;               /* [F,N,3] final image (renderer.py:390-397 / radnerf_torso.py:191-197) */
    float *depth_map;             /* [F,N] */
    float *weights_sum;           /* [F,N] head alpha */
    float *torso_alpha_map;       /* [F,N]   or NULL */
    float *torso_rgb_map;         /* [F,N,3] or NULL (bg mixed with torso, radnerf_torso.py:187-189) */
    float *torso_deform;          /* [F,N,2] deformation for masked pixels, 0 elsewhere; or NULL */
    int32_t *stats;               /* [F,4] = {B_total, n_survivors, S_valid_samples, P_torso_pixels} or NULL */
    uint8_t *rgb_u8;              /* [F,N,3] the frame as the video writer wants it, (uint8)(int)(rgb * 255) of the clamped colour
                                   * (inference/genefacepp_infer.py:469,505), written by the epilogue kernel itself; or NULL.
                                   * rgb_map may be NULL when rgb_u8 is given (then no fp32 frame is written at all) */
    /* The frame's alpha matte, for compositing over something other than one static background.  With ws = weights_sum, image
     * the premultiplied head colour and ta, tc the torso alpha and colour (both 0 outside the torso mask and for head-only models):
     *   coverage               A = ws + (1 - ws) * ta
     *   premultiplied colour   P = clamp(image + (1 - ws) * (tc * ta), 0, 1)
     * fp32, rounded at the same sites as the composite.  Head-only models: A = ws, P = clamp(image).  P + (1 - A) * B is the
     * frame rendered with bg_color = B (up to fp32 rounding wherever that composite was not clamped); P is that frame's colour
     * for B = 0 bit for bit.  Both ignore bg_color, so a call may ask for the frame over bg_color and for the matte together. */
    float *alpha_map;             /* [F,N] A, or NULL */
    uint8_t *rgba_u8;             /* [F,N,4] 4-byte aligned, written as one 32-bit store per pixel: (uint8)(int)(P * 255) per colour
                                   * channel (the truncation of rgb_u8) and (uint8)(int)(A * 255) in the fourth byte; or NULL.
                                   * At least one of rgb_map, rgb_u8 and rgba_u8 must be given. */
} gfpp_outputs;

GFPP_API size_t gfpp_render_workspace_bytes(uint32_t n_frames, uint32_t n_rays, uint32_t max_steps);
/* Enqueue the whole clip (or one frame): pass-1 persistent head kernel, on-device round-schedule
 * replay, pass-2 for rays that outlive max_steps, torso + composite epilogue.  No host sync. */
GFPP_API int gfpp_render_frames(const gfpp_model *model, const gfpp_frames *frames, const gfpp_outputs *out,
                                void *workspace, size_t workspace_bytes, void *stream);
/* Diagnostics for bench.py's roofline leg: when enabled, gfpp_render_frames records CUDA events (on the launching
 * stream) around its three main kernels; gfpp_profile_read() waits for those events and returns the durations of the
 * most recent call in milliseconds: ms[0] = head pass 1, ms[1] = schedule + head pass 2, ms[2] = torso/composite epilogue. */
GFPP_API int gfpp_profile_enable(int on);
GFPP_API int gfpp_profile_read(float ms[4]);   /* ms[3] = everything before the head kernel (memset, torso biases, ray setup) */
/* optional: device buffer of 32 uint64 that the tensor-core head kernel fills with per-phase cycle totals (thread 0 of each
 * CTA; slot 31 = batches processed); NULL switches it off.  Diagnostics only. */
GFPP_API int gfpp_profile_phases(void *dev_u64x32);
/* Self-test of the wgmma plumbing (tile layouts, descriptors, MMA issue, accumulator fragment read-back) used by the tensor-core MLP:
 * out[128,N] = A[128,K] @ W[N,K]^T with 16-bit operands, fp32 accumulation.  K = 64*j (+16 if k16_tail), N in {16, 128, 144}
 * (the MMA widths the kernels use), K <= 144.  precision: 1 = fp16, 2 = bf16 hi/lo split (3 MMAs), 3 = bf16.  scratch: >= 6*18432 bytes. */
GFPP_API int gfpp_tc_selftest(const float *A, const float *W, uint32_t N, uint32_t K, int k16_tail, int precision,
                              void *scratch, float *out, void *stream);
/* Debug / test hook: write out the rays the fused path generates IN-KERNEL from poses + intrinsics (pixel centres, normalised,
 * rotated by c2w[:3,:3]: modules/radnerfs/utils.py:302-360), [F, img_h*img_w, 3] each, so that tests can measure their distance to
 * torch get_rays and hand exactly these rays to the oracle. */
GFPP_API int gfpp_debug_generate_rays(const float *poses_c2w, uint32_t n_frames, float fx, float fy, float cx, float cy,
                                      uint32_t img_h, uint32_t img_w, float *rays_o, float *rays_d, void *stream);
/* number of kernels the last gfpp_render_frames call on this thread launched */
GFPP_API int gfpp_last_launch_count(void);

/* ------------------------------------------------------------------ (C) super-resolution head of the SR checkpoints
 *
 * Replaces `Superresolution.forward` (modules/radnerfs/radnerf_sr.py:15-48; StyleGAN2 blocks of
 * modules/eg3ds/models/superresolution.py:159-257 and networks_stylegan2.py:286-475) for the 256 -> 512 head the
 * `with_sr` checkpoints carry (inference/genefacepp_infer.py:464-465,480-481 takes `sr_rgb_map`).  The network is
 * always run with the constant latent w = 1 (radnerf_sr.py:33-34), so the style modulation, the demodulation and the
 * [1,3,3,1] resampling filter are constants of the checkpoint: the caller folds them into plain GEMM matrices (fp32,
 * device) once -- genefaceplusplus_b200/superres.py::folded_weights documents the algebra -- and hands them over here:
 *   conv_in_w  block0.conv0  [27][128]     k-major, k = (ky*3+kx)*3 + ci
 *   conv0_w    block0.conv1  [128][1152]   k = (ky*3+kx)*128 + ci
 *   up_w       block1.conv0  [256][1152]   transposed stride-2 conv + FIR merged into four 3x3 phase kernels on the input
 *                                          grid, row = (py*2+px)*64 + co for output pixel (2y+py, 2x+px)
 *   conv1_w    block1.conv1  [64][576]     k = (ky*3+kx)*64 + ci
 *   bias[4]    conv biases (128, 128, 64, 64);  rgb_w[2] effective toRGB weights [3][128], [3][64];  rgb_b[2] [3]
 * Operands of the three tensor-core layers are rounded to fp16 (fp32 accumulation), as the reference's use_fp16 blocks do. */
typedef struct {
    const float *conv_in_w;
    const float *conv0_w;
    const float *up_w;
    const float *conv1_w;
    const float *bias[4];
    const float *rgb_w[2];
    const float *rgb_b[2];
} gfpp_sr_desc;

typedef struct gfpp_sr_model {
    uint64_t opaque[32];
} gfpp_sr_model;

GFPP_API size_t gfpp_sr_packed_bytes(void);
/* Repack on `stream` into `packed` (device, 1024-byte aligned, >= gfpp_sr_packed_bytes); the desc's tensors are copied and
 * may be freed once the stream has passed this call. */
GFPP_API int gfpp_sr_pack(const gfpp_sr_desc *desc, void *packed, size_t packed_bytes, gfpp_sr_model *model, void *stream);
GFPP_API size_t gfpp_sr_workspace_bytes(uint32_t n_frames, uint32_t in_res);
/* rgb_in [F, in_res*in_res, 3] fp32 in [0,1] (the layout gfpp_render_frames writes `rgb_map` in) -> out [F, 3, 2*in_res,
 * 2*in_res] fp32 (planar, as the reference returns it); clamp01 != 0 clamps it to [0,1] (every caller of the SR head does
 * that next: radnerf_sr.py:208).  noise[i]: per-layer noise planes ALREADY multiplied by the layer's noise_strength
 * (layers 0,1: in_res^2; layers 2,3: (2*in_res)^2), one plane shared by all frames (noise_mode 'const') or, with
 * noise_per_frame != 0, F consecutive planes ('random'); NULL entries / a NULL array mean no noise ('none').
 * in_res must be a multiple of 128 (256 in the reference).  Four kernel launches, no host sync, no allocation. */
GFPP_API int gfpp_sr_forward(const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in,
                             const float *const noise[4], uint32_t noise_per_frame, float *out, int clamp01, void *workspace,
                             size_t workspace_bytes, void *stream);
/* gfpp_sr_forward for the video writer: the same four launches and workspace, the result always clamped to [0,1], and the
 * last epilogue writes either or both of
 *   out     [F, 3, 2*in_res, 2*in_res] fp32 planar (bit-identical to gfpp_sr_forward with clamp01 = 1), NULL: not written;
 *   out_u8  [F, 2*in_res, 2*in_res, 3] uint8 interleaved (HWC, what video writers take), 4-byte aligned, NULL: not written;
 *           value (int)(x * 255) of the clamped fp32 x -- the driver's `(rgb * 255).int()` (genefacepp_infer.py:469, 505).
 * At least one of them must be given.  A uint8-only call writes a quarter of the bytes of the fp32 frames. */
GFPP_API int gfpp_sr_forward_video(const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in,
                                   const float *const noise[4], uint32_t noise_per_frame, float *out, uint8_t *out_u8,
                                   void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (C) torso field of the torso-SR checkpoints
 *
 * Replaces RADNeRFTorsowithSR.forward_torso + the composite of its render() (modules/radnerfs/radnerf_torso_sr.py:75-113,
 * 196-228): mask by grid_sample of density_grid_torso, the landmark-conditioned (and, `torso_head_aware`, head-colour-aware)
 * deformation + canonical torso field on the masked pixels, torso over background, head over both, clamp.  The head NeRF of
 * these checkpoints is the plain head field: render it with gfpp_render_frames (has_torso = 0, bg_color = zeros, so that
 * `rgb_map` is the premultiplied head colour and `weights_sum` its alpha) and hand both over here; the result feeds
 * gfpp_sr_forward.  Weights in the reference's nn.Linear layout [out, in], fp32 device pointers (state_dict tensors); the
 * grid table, density_grid_torso, the first deform / canonical layers and the code are BORROWED (per-frame folds read them). */
typedef struct {
    gfpp_grid_desc torso_grid;          /* 2-D tiled grid, 16 levels x 2 */
    const float *torso_deform_w[3];     /* (64,din) (64,64) (2,64); din = 42 + torso_code_dim + 126 (+ 16 if head_aware) */
    const float *torso_canon_w[3];      /* (32,32+din) (32,32) (4,32) */
    const float *torso_code;            /* [torso_code_dim] = torso_individual_codes[0] */
    uint32_t torso_code_dim;            /* 8 */
    int head_aware;                     /* hparams['torso_head_aware'] */
    const float *ha_w[3];               /* head_color_weights_encoder: (16,4) (32,16) (16,32) */
    const float *ha_b[3];               /* its biases: 16, 32, 16 */
    const float *density_grid_torso;    /* [grid_size^2] */
    uint32_t grid_size;
    float density_thresh_torso;         /* min(density_thresh_torso, mean_density_torso) as the reference evaluates it */
    float torso_shrink;
} gfpp_torso_sr_desc;

typedef struct gfpp_torso_sr_model {
    uint64_t opaque[128];
} gfpp_torso_sr_model;

typedef struct {
    uint32_t n_frames;            /* F */
    uint32_t n_rays;              /* N pixels per frame (256*256 in the reference) */
    const float *image;           /* [F,N,3] premultiplied head colour */
    const float *weights_sum;     /* [F,N]   head alpha */
    const float *lm68;            /* [F,136] 68 2-D landmarks per frame (points 5..11 = the jaw are used) */
    const float *bg_coords;       /* [N,2]   shared by all frames */
    const float *bg_color;        /* [N,3]   shared by all frames, or NULL => 1.0 */
} gfpp_torso_sr_frames;

GFPP_API size_t gfpp_torso_sr_packed_bytes(void);
GFPP_API int gfpp_torso_sr_pack(const gfpp_torso_sr_desc *desc, void *packed, size_t packed_bytes, gfpp_torso_sr_model *model,
                                void *stream);
GFPP_API size_t gfpp_torso_sr_workspace_bytes(uint32_t n_frames);
/* rgb_map [F,N,3] (required): the clamped composite; torso_alpha_map [F,N], torso_rgb_map [F,N,3] (torso over background),
 * torso_deform [F,N,2] (0 outside the mask), torso_pixels [F] (masked pixels per frame): optional, NULL to skip.
 * Two kernel launches, no host sync, no allocation. */
GFPP_API int gfpp_torso_sr_composite(const gfpp_torso_sr_model *model, const gfpp_torso_sr_frames *frames, float *rgb_map,
                                     float *torso_alpha_map, float *torso_rgb_map, float *torso_deform, int32_t *torso_pixels,
                                     void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (D) training-side ops (SURVEY.md 8(f) rank 4)
 *
 * Mirror, argument for argument (+ stream; grid offsets as a host pointer, as in (A)), the training-side pybind functions of
 * the reference's extensions, so that its own autograd wrappers (raymarching.py:184-344, grid.py:24-88) can bind them:
 *   gfpp_march_rays_train                <- raymarching.h:14 (raymarching.cu:352-533)
 *   gfpp_march_rays_train_backward       <- raymarching.h:15 (raymarching.cu:535-598)
 *   gfpp_composite_rays_train_forward    <- raymarching.h:16 (raymarching.cu:603-700)
 *   gfpp_composite_rays_train_backward   <- raymarching.h:17 (raymarching.cu:711-822)
 *   gfpp_grid_encode_forward_dydx        <- gridencoder.h:12 with dy_dx given (gridencoder.cu:87-243)
 *   gfpp_grid_encode_backward            <- gridencoder.h:13 (gridencoder.cu:246-368, 413-443)
 *   gfpp_grad_total_variation            <- gridencoder.h:15 (gridencoder.cu:505-609)
 *   gfpp_packbits / gfpp_morton3D / gfpp_morton3D_invert / gfpp_morton3D_dilation / gfpp_sph_from_ray
 *                                        <- raymarching.h:8-12 (raymarching.cu:162-342; update_extra_state)
 * fp32 only.  One deliberate difference: gfpp_march_rays_train is deterministic -- point offsets are an exclusive prefix sum of
 * the per-ray sample counts in ray order (rays[n] = (n, offset, num_steps)) instead of the reference's atomicAdd arrival
 * order; every consumer addresses samples through `rays`, so this is one of the layouts the reference itself can produce.
 * It needs a small scratch buffer for the device-wide scan (query the size first).  `counter` keeps the reference's
 * meaning: counter[0] += points, counter[1] += N. */
GFPP_API size_t gfpp_march_rays_train_scratch_bytes(uint32_t N);
GFPP_API int gfpp_march_rays_train(const float *rays_o, const float *rays_d, const uint8_t *grid, float bound, float dt_gamma,
                                   uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float *nears,
                                   const float *fars, float *xyzs, float *dirs, float *deltas, int32_t *rays, int32_t *counter,
                                   const float *noises, void *scratch, size_t scratch_bytes, void *stream);
/* grad_rays_o / grad_rays_d [N,3] are accumulated into (+=), as in the reference */
GFPP_API int gfpp_march_rays_train_backward(const float *grad_xyzs, const float *grad_dirs, const int32_t *rays, const float *deltas,
                                            uint32_t N, uint32_t M, float *grad_rays_o, float *grad_rays_d, void *stream);
GFPP_API int gfpp_composite_rays_train_forward(const float *sigmas, const float *rgbs, const float *ambient, const float *deltas,
                                               const int32_t *rays, uint32_t M, uint32_t N, float T_thresh, float *weights_sum,
                                               float *ambient_sum, float *depth, float *image, void *stream);
/* grad_sigmas [M], grad_rgbs [M,3], grad_ambient [M] must be zero-initialised by the caller (raymarching.py:316-318) */
GFPP_API int gfpp_composite_rays_train_backward(const float *grad_weights_sum, const float *grad_ambient_sum, const float *grad_image,
                                                const float *sigmas, const float *rgbs, const float *ambient, const float *deltas,
                                                const int32_t *rays, const float *weights_sum, const float *ambient_sum,
                                                const float *image, uint32_t M, uint32_t N, float T_thresh, float *grad_sigmas,
                                                float *grad_rgbs, float *grad_ambient, void *stream);
/* outputs [L,B,C] as gfpp_grid_encode_forward, plus dy_dx [B, L, D, C] */
GFPP_API int gfpp_grid_encode_forward_dydx(const float *inputs, const float *embeddings, const int32_t *offsets_host, float *outputs,
                                           uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, float *dy_dx,
                                           uint32_t gridtype, int align_corners, uint32_t interp, void *stream);
/* grad [L,B,C]; grad_embeddings (zero-initialised by the caller, grid.py:76) is accumulated into with vector reductions;
 * dy_dx / grad_inputs [B,D]: both or neither */
GFPP_API int gfpp_grid_encode_backward(const float *grad, const float *inputs, const float *embeddings, const int32_t *offsets_host,
                                       float *grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
                                       const float *dy_dx, float *grad_inputs, uint32_t gridtype, int align_corners, uint32_t interp,
                                       void *stream);
GFPP_API int gfpp_grad_total_variation(const float *inputs, const float *embeddings, float *grad, const int32_t *offsets_host,
                                       float weight, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
                                       uint32_t gridtype, int align_corners, void *stream);
GFPP_API int gfpp_packbits(const float *grid, uint32_t N, float density_thresh, uint8_t *bitfield, void *stream);
GFPP_API int gfpp_morton3D(const int32_t *coords, uint32_t N, int32_t *indices, void *stream);
GFPP_API int gfpp_morton3D_invert(const int32_t *indices, uint32_t N, int32_t *coords, void *stream);
GFPP_API int gfpp_morton3D_dilation(const float *grid, uint32_t C, uint32_t H, float *grid_dilation, void *stream);
GFPP_API int gfpp_sph_from_ray(const float *rays_o, const float *rays_d, float radius, uint32_t N, float *coords, void *stream);

/* ------------------------------------------------------------------ (E) occupancy-grid maintenance (SURVEY.md 8(f) rank 4)
 *
 * The head model's density grid as NeRFRenderer maintains it during training (modules/radnerfs/renderer.py:131-278), on a
 * packed model.  The density query evaluates the head field up to the sigma net (RADNeRF.density, radnerf.py:143-166) in the
 * arithmetic of the model's mode: fp16 models on wgmma with their fp16 operand images and fp16 tables (what they render); fp32,
 * bf16x3, bf16 and robust models with the fp32 weight chunks and fp32 tables.  Everything is enqueued on `stream` with
 * no host synchronisation and no allocation, and is bit-identical from run to run (no atomics whose order reaches an output).
 *
 * gfpp_density_query: sigma [n] = trunc_exp(h0) (raw: density_scale is NOT applied, as in density()); geo_feat [n,128] = h[1:129]
 *   or NULL.  xyzs [n,3] in [-bound, bound]; cond_feat [64].  cond_feat and geo_feat 16-byte aligned.
 * gfpp_density_grid_update: update_extra_state's grid refresh (renderer.py:230-278) --
 *   1. sigma * density_scale at every cell of every cascade into tmp [C, H^3] (Morton order), the cell positions computed from
 *      noise [C,H,H,H,3] in [0,1) (the rand_like draws of renderer.py:258 in meshgrid(x,y,z) order) in fp32 exactly as the reference;
 *   2. tmp = 6-neighbour dilation; where density_grid >= 0 and tmp >= 0: density_grid = max(density_grid * decay, tmp);
 *   3. *mean_out = mean(clamp(density_grid, 0)) (double accumulation, fixed order; device scalar);
 *   4. the model's bitfield = packbits(density_grid, min(*mean_out, density_thresh)), threshold read on the device;
 *   5. the packed model's occupied-cell bounds and coarse occupancy are rebuilt in place: the next gfpp_render_frames on `model`
 *      marches the new grid without a repack.
 *   density_grid [C, H^3] (16-byte aligned) is updated in place; tmp_grid [C, H^3] receives the raw (pre-dilation) densities, or
 *   NULL.  The bitfield is written on `stream`: a render that reads it on another stream must be ordered against this call.
 *   Cascade and grid_size come from the model: cascade 1..8, grid_size a power of two in 8..512 (Morton codes below H^3 cover
 *   the grid only then); workspace: gfpp_density_grid_workspace_bytes (0 = unsupported shape).
 * gfpp_mark_untrained_grid: mark_untrained_grid (renderer.py:131-199): density_grid [C, H^3] cells that no camera of
 *   poses_c2w [B,4,4] sees are set to -1, the others are left as they are.  Intrinsics and bound as the reference's Python
 *   floats (double); the coverage test runs in fp32 in the reference's operation order. */
GFPP_API int gfpp_density_query(const gfpp_model *model, const float *xyzs, uint32_t n, const float *cond_feat, float *sigma,
                                float *geo_feat, void *stream);
GFPP_API size_t gfpp_density_grid_workspace_bytes(uint32_t cascade, uint32_t grid_size);
GFPP_API int gfpp_density_grid_update(const gfpp_model *model, const float *cond_feat, const float *noise, float decay,
                                      float density_thresh, float *density_grid, float *mean_out, float *tmp_grid, void *workspace,
                                      size_t workspace_bytes, void *stream);
GFPP_API int gfpp_mark_untrained_grid(const float *poses_c2w, uint32_t n_poses, double fx, double fy, double cx, double cy,
                                      double bound, uint32_t cascade, uint32_t grid_size, float *density_grid, void *stream);

/* ------------------------------------------------------------------ (F) torso occupancy grid (SURVEY.md 8(f) rank 4)
 *
 * density_grid_torso [H*H] as the torso models maintain it during training (RADNeRFTorso.update_extra_state,
 * radnerf_torso.py:201-242; RADNeRFTorsowithSR.update_extra_state, radnerf_torso_sr.py:246-288), H = the packed model's
 * grid_size in 2..4096.  The torso fields run in fp32 FFMA, in the arithmetic of the render epilogues.  Everything is enqueued
 * on `stream` with no host synchronisation and no allocation, and is bit-identical from run to run.  `code` is one row of
 * torso_individual_codes [torso_code_dim] (the refresh uses row rand_idx, not row 0); it is NULL iff torso_code_dim == 0.
 * Workspaces: gfpp_torso_grid_workspace_bytes(grid_size) for the refresh (0 = unsupported size), gfpp_torso_query_workspace_bytes()
 * for the query (the two folded bias vectors only; a refresh workspace is large enough for it too).
 *
 * gfpp_torso_query: forward_torso (radnerf_torso.py:51-84) of a model packed with has_torso = 1 at xy [n,2] in [-1,1] for the
 *   head pose pose6 [6] (convert_poses): alpha [n], color [n,3] or NULL, deform [n,2] (dx before the clamp) or NULL.
 * gfpp_torso_grid_update / gfpp_torso_sr_grid_update: the refresh, for the plain torso model (pose6 [6]) and for the torso-SR
 *   model (lm68 [136]; with head_aware its encoder sees image = weights_sum = 0, as the reference passes it) --
 *   1. alpha at every cell into tmp [H*H] at the reference's transposed index y*H + x, the cell positions computed from
 *      noise [H,H,2] in [0,1) (the rand_like draws in meshgrid(x, y) order) in fp32 exactly as the reference;
 *   2. tmp = 5x5 max (max_pool2d, stride 1, padding 2); density_grid_torso = max(density_grid_torso * decay, tmp) in place;
 *   3. *mean_out = mean(density_grid_torso) (no clamp; double accumulation, fixed order; device scalar).
 *   tmp_grid [H*H] receives the raw (pre-dilation) alphas, or NULL.
 * gfpp_model_set_torso_threshold / gfpp_torso_sr_set_threshold: host-only write of the mask threshold
 *   min(density_thresh_torso, mean_density_torso) into the handle: the next render masks with it without a repack. */
GFPP_API size_t gfpp_torso_grid_workspace_bytes(uint32_t grid_size);
GFPP_API size_t gfpp_torso_query_workspace_bytes(void);
GFPP_API int gfpp_torso_query(const gfpp_model *model, const float *xy, uint32_t n, const float *pose6, const float *code,
                              float *alpha, float *color, float *deform, void *workspace, size_t workspace_bytes, void *stream);
GFPP_API int gfpp_torso_grid_update(const gfpp_model *model, const float *pose6, const float *code, const float *noise,
                                    float decay, float *density_grid_torso, float *mean_out, float *tmp_grid, void *workspace,
                                    size_t workspace_bytes, void *stream);
GFPP_API int gfpp_torso_sr_grid_update(const gfpp_torso_sr_model *model, const float *lm68, const float *code, const float *noise,
                                       float decay, float *density_grid_torso, float *mean_out, float *tmp_grid, void *workspace,
                                       size_t workspace_bytes, void *stream);
GFPP_API int gfpp_model_set_torso_threshold(gfpp_model *model, float density_thresh_torso);
GFPP_API int gfpp_torso_sr_set_threshold(gfpp_torso_sr_model *model, float density_thresh_torso);

/* ------------------------------------------------------------------ (G) trainable head field
 *
 * RADNeRF.forward (modules/radnerfs/radnerf.py:108-141) and its gradient for the training step, in fp32 FFMA arithmetic (the
 * reference's amp: false), reading the parameters IN PLACE through a gfpp_model_desc -- no gfpp_model_pack: the weights change
 * after every optimizer step.  Read from the desc: both grids (reference layout [entries,2] fp32, 8-byte aligned; 16 levels x 2;
 * position 3-D, ambient 2-D or 3-D), the eight nn.Linear weights [out, in] (16-byte aligned; the May shapes of gfpp_model_pack),
 * individual_code [ind_dim] (the training row individual_embeddings[index]; NULL iff ind_dim == 0; ind_dim 0, 4, 8, 12 or 16),
 * cond_dim (64), bound and mlp_precision (must be 0).  Anything else returns GFPP_ERR_UNSUPPORTED or GFPP_ERR_INVALID.  The other
 * desc fields are not read.  Every argument is validated before any CUDA call; M == 0 then returns GFPP_OK without touching the
 * device (the data pointers may be NULL).  Everything is enqueued on `stream` with no host synchronisation and no allocation.
 *
 * Workspace (256-byte aligned): gfpp_field_backward_workspace_bytes(M) for the backward (0 = unsupported M); the forward needs
 * gfpp_field_backward_workspace_bytes(0) bytes (the per-call k-major copy of the weights, ~320 KB), so a backward workspace fits both.
 *
 * gfpp_field_forward: for points xyzs [M,3] in [-bound, bound], dirs [M,3], one cond_feat [64]:
 *   sigma [M] = exp(h0) raw (density_scale is the caller's, renderer.py:376), color [M,3] (sigmoid), ambient_pos [M,A] (tanh).
 * gfpp_field_backward: given grad_sigma [M] (w.r.t. the raw sigma), grad_color [M,3] and grad_ambient_pos [M,A] (the ambient
 *   regulariser's gradient enters there), recomputes the forward and writes
 *     grad_w[0..7]  the gradients of ambient_w[0..2], sigma_w[0..2], color_w[0..1], same [out, in] layout (overwritten);
 *     grad_cond [64] (cond_feat is repeated over the points: its gradient is the sum), grad_code [ind_dim] (NULL iff ind_dim == 0);
 *     grad_position_table / grad_ambient_table [entries,2]: ACCUMULATED into (+=), as the reference's grid backward does.
 *   trunc_exp' = exp(clamp(h0, -15, 15)); the ambient grid's input gradient goes through its dy_dx and the (x+1)/2 map of bound 1;
 *   the position grid gets no input gradient (xyzs never requires grad in the reference).
 * Determinism: the forward outputs, grad_w, grad_cond and grad_code are bit-identical from run to run (per-CTA partial sums in the
 * workspace, reduced in a fixed order by one kernel; the partitioning depends only on M).  The two table gradients are scattered
 * with float2 vector reductions, so their summation order is free. */
GFPP_API size_t gfpp_field_backward_workspace_bytes(uint32_t M);
GFPP_API int gfpp_field_forward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat,
                                float *sigma, float *color, float *ambient_pos, void *workspace, size_t workspace_bytes, void *stream);
GFPP_API int gfpp_field_backward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat,
                                 const float *grad_sigma, const float *grad_color, const float *grad_ambient_pos, float *const grad_w[8],
                                 float *grad_cond, float *grad_code, float *grad_position_table, float *grad_ambient_table, void *workspace,
                                 size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (H) trainable torso field
 *
 * RADNeRFTorso.forward_torso (modules/radnerfs/radnerf_torso.py:51-84) and its gradient for the torso training step, in fp32 FFMA
 * arithmetic, reading the parameters IN PLACE through a gfpp_model_desc -- no gfpp_model_pack.  Read from the desc: torso_grid
 * (2-D, 16 levels x 2, reference layout [entries,2] fp32, 8-byte aligned), torso_deform_w (64,din) (64,64) (2,64), torso_canon_w
 * (32,32+din) (32,32) (4,32) with din = 42 + 54 + torso_code_dim, torso_code_dim (<= 10) and torso_shrink.  The other desc fields
 * are not read (has_torso and torso_code neither: `code` is an explicit argument, the training row torso_individual_codes[index];
 * it is NULL iff torso_code_dim == 0).  pose6 [6] is the head pose (convert_poses).  Every argument is validated before any CUDA
 * call; M == 0 then returns GFPP_OK without touching the device (the point and output pointers may be NULL).  Everything is enqueued
 * on `stream` with no host synchronisation and no allocation.
 *
 * Workspace (256-byte aligned): gfpp_torso_field_workspace_bytes(M) for the backward (0 = unsupported M); the forward needs
 * gfpp_torso_field_workspace_bytes(0) bytes (the per-call k-major copy of the weights and the two folded bias vectors, ~42 KB).
 *
 * gfpp_torso_field_forward: for points xy [M,2] in [-1,1]: alpha [M], color [M,3] (sigmoid), deform [M,2] (dx, before the clamp).
 *   Bit-identical to gfpp_torso_query of a model packed from the same parameters, with the same pose6 and code.
 * gfpp_torso_field_backward: given grad_alpha [M], grad_color [M,3] and grad_deform [M,2] (w.r.t. dx), recomputes the forward and
 *   writes grad_deform_w[0..2], grad_canon_w[0..2] (same [out, in] layouts; overwritten) and grad_code [torso_code_dim] (the code
 *   is repeated over the points: its gradient is the sum; NULL iff torso_code_dim == 0); grad_torso_table [entries,2] is
 *   ACCUMULATED into (+=), as the reference's grid backward does.  The grid's input gradient goes through its dy_dx, the (x+1)/2
 *   map of bound 1 and the clamp (which passes the gradient on [-1, 1] inclusive); the pose gets no gradient, xy neither.
 * Determinism: the forward outputs, grad_deform_w, grad_canon_w and grad_code are bit-identical from run to run (per-CTA partial
 * sums in the workspace, reduced in a fixed order by one kernel; the partitioning depends only on M).  The table gradient is
 * scattered with float2 vector reductions, so its summation order is free. */
GFPP_API size_t gfpp_torso_field_workspace_bytes(uint32_t M);
GFPP_API int gfpp_torso_field_forward(const gfpp_model_desc *desc, const float *xy, uint32_t M, const float *pose6, const float *code,
                                      float *alpha, float *color, float *deform, void *workspace, size_t workspace_bytes, void *stream);
GFPP_API int gfpp_torso_field_backward(const gfpp_model_desc *desc, const float *xy, uint32_t M, const float *pose6, const float *code,
                                       const float *grad_alpha, const float *grad_color, const float *grad_deform,
                                       float *const grad_deform_w[3], float *const grad_canon_w[3], float *grad_code,
                                       float *grad_torso_table, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (I) trainable torso-SR field
 *
 * RADNeRFTorsowithSR.forward_torso (modules/radnerfs/radnerf_torso_sr.py:75-114) and its gradient for the torso training step
 * (on_train_torso_nerf), in fp32 FFMA arithmetic, reading the parameters IN PLACE through a gfpp_torso_sr_desc -- no
 * gfpp_torso_sr_pack.  Read from the desc: torso_grid (2-D, 16 levels x 2, reference layout [entries,2] fp32, 8-byte aligned),
 * torso_deform_w (64,din) (64,64) (2,64), torso_canon_w (32,32+din) (32,32) (4,32) with din = 42 + torso_code_dim + 126 (+ 16 with
 * head_aware), torso_code_dim (<= 10), head_aware, ha_w / ha_b (head_color_weights_encoder (16,4) (32,16) (16,32) and its biases;
 * read iff head_aware) and torso_shrink.  The other desc fields are not read (torso_code neither: `code` is an explicit argument,
 * the training row torso_individual_codes[index]; it is NULL iff torso_code_dim == 0).  lm68 [136] are the frame's landmarks
 * (points 5..11 are used).  image [M,3] and weights_sum [M] are the head colour and alpha at the points that the head-aware encoder
 * sees; both NULL means zeros (the reference's image=None path).  Passing only one of them, or passing them without head_aware, is
 * invalid.  Every argument is validated before any CUDA call; M == 0 then returns GFPP_OK without touching the device (the point
 * and output pointers may be NULL).  Everything is enqueued on `stream` with no host synchronisation and no allocation.
 *
 * Workspace (256-byte aligned): gfpp_torso_sr_field_workspace_bytes(M) for the backward (0 = unsupported M); the forward needs
 * gfpp_torso_sr_field_workspace_bytes(0) bytes (the per-call k-major copy of the weights and the encoder and the two folded bias
 * vectors, ~52 KB).
 *
 * gfpp_torso_sr_field_forward: for points xy [M,2] in [-1,1]: alpha [M], color [M,3] (sigmoid), deform [M,2] (dx, before the clamp).
 *   It is the render epilogue's own field code (k_torso_sr) on these points: bit-identical to gfpp_torso_sr_composite's
 *   torso_alpha_map and torso_deform at its masked pixels, for the same parameters, code, lm68, image and weights_sum.
 * gfpp_torso_sr_field_backward: given grad_alpha [M], grad_color [M,3] and grad_deform [M,2] (w.r.t. dx), recomputes the forward and
 *   writes grad_deform_w[0..2], grad_canon_w[0..2], grad_ha_w[0..2], grad_ha_b[0..2] (same layouts as the parameters; overwritten;
 *   the grad_ha_* arrays are NULL iff head_aware == 0) and grad_code [torso_code_dim] (the code is repeated over the points: its
 *   gradient is the sum; NULL iff torso_code_dim == 0); grad_torso_table [entries,2] is ACCUMULATED into (+=), as the reference's grid
 *   backward does.  The grid's input gradient goes through its dy_dx, the (x+1)/2 map of bound 1 and the clamp (which passes the
 *   gradient on [-1, 1] inclusive); the head-aware encoding's gradient is the sum over both first layers' encoding columns, then
 *   through the encoder (LeakyReLU slope 0.02 where its output is <= 0).  lm68, xy, image and weights_sum get no gradient.
 * Determinism: the forward outputs and every gradient except the table's are bit-identical from run to run (per-CTA partial sums in
 * the workspace, reduced in a fixed order by one kernel; the partitioning depends only on M).  The table gradient is scattered with
 * float2 vector reductions, so its summation order is free. */
GFPP_API size_t gfpp_torso_sr_field_workspace_bytes(uint32_t M);
GFPP_API int gfpp_torso_sr_field_forward(const gfpp_torso_sr_desc *desc, const float *xy, uint32_t M, const float *lm68, const float *code,
                                         const float *image, const float *weights_sum, float *alpha, float *color, float *deform,
                                         void *workspace, size_t workspace_bytes, void *stream);
GFPP_API int gfpp_torso_sr_field_backward(const gfpp_torso_sr_desc *desc, const float *xy, uint32_t M, const float *lm68, const float *code,
                                          const float *image, const float *weights_sum, const float *grad_alpha, const float *grad_color,
                                          const float *grad_deform, float *const grad_deform_w[3], float *const grad_canon_w[3],
                                          float *const grad_ha_w[3], float *const grad_ha_b[3], float *grad_code, float *grad_torso_table,
                                          void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (J) trainable head field on tensor cores
 *
 * The functions of (G) in a second arithmetic: the six 128-wide layers run as fp16 wgmma products with fp32 accumulation, forward
 * and backward (input gradients against transposed fp16 weight images, weight gradients as dY^T X over 128-point tiles).  The
 * parameters are read in place as fp32 and are not rounded in memory; all gradients come out in fp32.  Rounded to fp16: the
 * operands of those products only (grid features, SH, hidden activations, weights, output gradients).  The grid gathers and
 * scatters, biases, activation functions and their derivatives and the three narrow layers (ambient logits, the sigma row, colour
 * logits) are fp32, the narrow layers on the fp32 accumulators -- the inputs of tanh and exp are never rounded to 16 bits.
 * Every block of output gradients is scaled by a power of two taken from its largest magnitude before it is rounded and the product
 * is scaled back in fp32, so upstream gradients multiplied by 2^k (loss scaling) give the same gradients times 2^k, and tiny
 * upstream gradients are not flushed to zero.
 *
 * Arguments, desc fields read, validation, status codes, M == 0, gradient targets (grad_w overwritten, table gradients accumulated)
 * and determinism are those of gfpp_field_forward / gfpp_field_backward; mlp_precision must be 0 here too (it names the inference
 * arithmetic).  Results differ from (G) by the fp16 rounding: about 1e-3 absolute on colour and ambient_pos.
 * Workspace (256-byte aligned): gfpp_field_tc_workspace_bytes(M) for the backward (0 = unsupported M); the forward needs
 * gfpp_field_tc_workspace_bytes(0) bytes (the per-call fp16 weight images, ~340 KB). */
GFPP_API size_t gfpp_field_tc_workspace_bytes(uint32_t M);
GFPP_API int gfpp_field_tc_forward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat,
                                   float *sigma, float *color, float *ambient_pos, void *workspace, size_t workspace_bytes, void *stream);
GFPP_API int gfpp_field_tc_backward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat,
                                    const float *grad_sigma, const float *grad_color, const float *grad_ambient_pos, float *const grad_w[8],
                                    float *grad_cond, float *grad_code, float *grad_position_table, float *grad_ambient_table,
                                    void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (K) frozen head of the torso training steps
 *
 * The no-grad head block of the torso training step (radnerf_torso.py:92-150 and radnerf_torso_sr.py:150 under torch.no_grad):
 * near_far_from_aabb + march_rays_train + RADNeRF.forward + composite_rays_train in one pass over the packed head model of
 * gfpp_model_pack, for one frame of N rays.  It runs k_ray_setup and pass 1 of the head kernel of the model's mlp_precision, with
 * composite_rays_train's termination: T is the running product of (1 - alpha), a ray stops after the sample that takes T below
 * T_thresh, after max_steps samples, or when it leaves the volume.  Nothing is written to HBM per sample and the host is never
 * synchronised.  Rays are slab-tested against the per-call `aabb` (host, xmin ymin zmin xmax ymax zmax; the torso steps pass
 * aabb_train) with the model's min_near.  cond_feat: device [64].  code: device [ind_dim], the training row of
 * individual_embeddings, folded into a copy of the colour-L0 bias in the workspace (the packed model is not written), or NULL;
 * it must be given iff the model was packed with ind_dim > 0.  noises: device [N] in [0,1), march_rays_train's jittered starts
 * (near + clamp(near * dt_gamma, dt_min, dt_max) * noise), or NULL for none.  Outputs: weights_sum [N] and the premultiplied head
 * image [N,3] (before any background) -- composite_rays_train's first and fourth outputs; rays that miss the volume get zeros.
 * There is no ambient_sum and no depth.  The sample budget of march_rays_train with mean_count > 0 is not modelled: every ray
 * gets up to max_steps samples (force_all_rays).
 * Validation (before any CUDA call): NULL pointers, a model handle not filled by gfpp_model_pack, N == 0, max_steps outside
 * 1..4096, code given iff ind_dim > 0, aabb with min > max, a workspace below gfpp_frozen_head_workspace_bytes(N, max_steps)
 * or not 256-byte aligned.  Stream-ordered, no host sync, deterministic.
 * gfpp_frozen_head_workspace_bytes returns 0 for N == 0, N >= 2^31 or max_steps outside 1..4096. */
GFPP_API size_t gfpp_frozen_head_workspace_bytes(uint32_t N, uint32_t max_steps);
GFPP_API int gfpp_frozen_head(const gfpp_model *model, const float *rays_o, const float *rays_d, uint32_t N, const float aabb[6],
                              const float *cond_feat, const float *code, const float *noises, float dt_gamma, uint32_t max_steps,
                              float T_thresh, float *weights_sum, float *image, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------ (L) grid encoder on half tables
 *
 * The grid encoder's ops of (A) and (D) on IEEE binary16 tables, as the reference runs them under autocast (grid.py:41-44 casts
 * tables with an even C to half): its scalar_t = at::Half instantiations of gridencoder.cu:87-368, argument for argument.  Every
 * 16-bit buffer is a uint16_t array of binary16 bit patterns (embeddings, outputs, dy_dx, grad, grad_embeddings, grad_inputs),
 * 4-byte aligned; inputs stay fp32 [B,D] in [0,1] and offsets_host is a HOST pointer as in (A).  C == 2, D in {2,3}, L <= 16.
 * The arithmetic is the reference's: fp32 weights, a half running sum per output (each corner's term rounded to half, then the
 * sum rounded to half, in the reference's corner order), the level constants from the device exp2f (scale = exp2f(level*S)*H - 1,
 * unlike the host-side scale of the fp32 ops), round-to-nearest-even at every rounding site.
 *
 * gfpp_grid_encode_forward_half: outputs [L,B,2]; dy_dx [B,L,D,2] or NULL (calc_grad_inputs).  Inputs outside [0,1] give zeros.
 * gfpp_grid_encode_backward_half: grad [L,B,2]; grad_embeddings [entries,2] (zero-initialised by the caller, grid.py:76) is
 *   accumulated into with one f16x2 vector reduction (red.global.add.noftz.f16x2) per corner: each add rounds to half and the
 *   order of the adds is free, as in the reference.  dy_dx [B,L,D,2] and grad_inputs [B,D]: both or neither; grad_inputs is
 *   overwritten with the half running sum over (level, channel) of the half products grad * dy_dx.
 * Validation (before any CUDA call): NULL pointers and dy_dx without grad_inputs -> GFPP_ERR_INVALID; C != 2, D outside {2,3},
 * L outside 1..16 or an empty level -> GFPP_ERR_UNSUPPORTED; a 16-bit pair buffer not 4-byte aligned -> GFPP_ERR_INVALID.
 * B == 0 returns GFPP_OK without touching the device. */
GFPP_API int gfpp_grid_encode_forward_half(const float *inputs, const uint16_t *embeddings, const int32_t *offsets_host, uint16_t *outputs,
                                           uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, uint16_t *dy_dx,
                                           uint32_t gridtype, int align_corners, uint32_t interp, void *stream);
GFPP_API int gfpp_grid_encode_backward_half(const uint16_t *grad, const float *inputs, const uint16_t *embeddings, const int32_t *offsets_host,
                                            uint16_t *grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
                                            const uint16_t *dy_dx, uint16_t *grad_inputs, uint32_t gridtype, int align_corners,
                                            uint32_t interp, void *stream);

/* ------------------------------------------------------------------ (M) torso pass of the torso training steps
 *
 * The per-pixel code between the frozen head (K) and the torso fields (H) / (I) in the torso training steps of both torso models
 * (radnerf_torso.py:165-193, radnerf_torso_sr.py:196-221): the grid_sample mask of density_grid_torso, the compaction of the
 * masked pixels, and the three-way composite forward and backward.  The entry points take the grid and plain arrays, no model
 * descriptor; the fields run unchanged on the compacted points with a host M.  A step is: gfpp_torso_mask, one read of *count,
 * the field's forward, gfpp_torso_composite_forward; then gfpp_torso_composite_backward and the field's backward.
 *
 * gfpp_torso_mask: pixel i of bg_coords [N,2] (8-byte aligned) is masked iff grid_sample(density_grid_torso [G,G], bg_coords[i],
 *   align_corners=True, bilinear, zeros padding) > thr, in ATen's grid_sampler_2d arithmetic.  thr is the fp32 value of
 *   min(density_thresh_torso, mean_density_torso): PyTorch compares a float32 tensor with a Python float scalar in float32, so the
 *   double is rounded to the nearest float first (what a C float argument does).  Outputs, with M the number of masked pixels:
 *     idx [N] (first M written): the masked pixel indices in ascending order -- the order of bg_coords[mask];
 *     slot [N]: the compacted row of each pixel, or -1;  xy [M,2] (8-byte aligned) = bg_coords[mask];
 *     image_m [M,3] = image[mask] and weights_sum_m [M] = weights_sum[mask]: the SR field's head-aware inputs, all four of image
 *       [N,3], weights_sum [N], image_m and weights_sum_m given, or all NULL;
 *     *count = M (device int32).
 *   Three launches (tile counts, a one-CTA scan of the counts, a tile-local scan that writes); no atomics, so every output is
 *   bit-identical from run to run.  Workspace: gfpp_torso_pass_workspace_bytes(N), 256-byte aligned (the tile counts).
 * gfpp_torso_composite_forward: one thread per pixel; a = alpha[slot[i]] and c = color[slot[i]] (alpha [M], color [M,3]; 0 where
 *   slot is -1; both may be NULL iff M == 0), bg the scalar 1 (bg_mode 0, bg_color NULL: bg_color=None), one colour (bg_mode 1,
 *   bg_color [3]) or one colour per pixel (bg_mode 2, bg_color [N,3]):
 *     torso_alpha_map [N] = a;  torso_rgb_map [N,3] = c*a + bg*(1-a);  rgb_map [N,3] = clamp(image + (1-weights_sum)*torso_rgb_map, 0, 1)
 *   in PyTorch's op order with every product and sum rounded separately: bit-identical to the composed recipe (zeros, index_put,
 *   the composite and the clamp in eager PyTorch).
 * gfpp_torso_composite_backward: one thread per masked point j < M, pixel idx[j]: given the upstream gradients of torso_alpha_map
 *   [N], torso_rgb_map [N,3] and rgb_map [N,3] (each may be NULL: zero), writes grad_alpha [M] and grad_color [M,3], the inputs of
 *   the fields' backward.  The clamp passes the gradient where 0 <= x <= 1 (torch.clamp), x recomputed with the forward's
 *   arithmetic.  M == 0 returns GFPP_OK without touching the device (idx and the gradient pointers may then be NULL).
 * Validation (before any CUDA call): NULL pointers, N == 0 -> GFPP_ERR_INVALID; N >= 2^31, G outside 2..4096 ->
 * GFPP_ERR_UNSUPPORTED; M > N, bg_mode outside 0..2 or bg_color given iff bg_mode == 0 -> GFPP_ERR_INVALID; a workspace below
 * gfpp_torso_pass_workspace_bytes(N) -> GFPP_ERR_WORKSPACE, or not 256-byte aligned -> GFPP_ERR_INVALID.  Stream-ordered, no host
 * sync, no allocation.  gfpp_torso_pass_workspace_bytes returns 0 for N == 0 or N >= 2^31. */
GFPP_API size_t gfpp_torso_pass_workspace_bytes(uint32_t N);
GFPP_API int gfpp_torso_mask(const float *density_grid_torso, uint32_t G, float thr, const float *bg_coords, uint32_t N, const float *image,
                             const float *weights_sum, int32_t *idx, int32_t *slot, float *xy, float *image_m, float *weights_sum_m,
                             int32_t *count, void *workspace, size_t workspace_bytes, void *stream);
GFPP_API int gfpp_torso_composite_forward(const int32_t *slot, uint32_t N, uint32_t M, const float *alpha, const float *color,
                                          const float *image, const float *weights_sum, const float *bg_color, uint32_t bg_mode,
                                          float *torso_alpha_map, float *torso_rgb_map, float *rgb_map, void *stream);
GFPP_API int gfpp_torso_composite_backward(const int32_t *idx, uint32_t N, uint32_t M, const float *alpha, const float *color,
                                           const float *image, const float *weights_sum, const float *bg_color, uint32_t bg_mode,
                                           const float *grad_torso_alpha_map, const float *grad_torso_rgb_map, const float *grad_rgb_map,
                                           float *grad_alpha, float *grad_color, void *stream);

/* ------------------------------------------------------------------ (N) planar I420 video frames
 *
 * gfpp_rgb_u8_to_i420 converts F interleaved uint8 RGB frames rgb [F,H,W,3] (the rgb_u8 frames of gfpp_render_frames, the video
 * frames of gfpp_sr_forward_video) to F planar yuv420p frames, ffmpeg's rawvideo layout, one after the other in out:
 *   frame f at out + f*H*W*3/2:  Y [H,W], then U [H/2,W/2], then V [H/2,W/2].
 * BT.601 limited range in integer arithmetic (>> is an arithmetic shift, i.e. floor division by 256):
 *   Y = ((66 R + 129 G + 25 B + 128) >> 8) + 16                          per pixel, 16..235
 *   R', G', B' = (sum of the 2x2 block's four values + 2) >> 2           per 2x2 block and channel (box average)
 *   U = ((-38 R' - 74 G' + 112 B' + 128) >> 8) + 128                     per 2x2 block, 16..240
 *   V = ((112 R' - 94 G' - 18 B' + 128) >> 8) + 128
 * The chroma of a block is its box average, so it is sited at the centre of its four luma samples (MPEG-1 / JPEG siting, not the
 * left siting that H.264 decoders assume by default).  The bytes are not those of ffmpeg's swscale conversion, whose rounding and
 * chroma filter differ.  rgb and out must not overlap.  Rows whose width is a multiple of 4 with both buffers 4-byte aligned are
 * read and written with 32-bit accesses; any other even width or alignment takes a byte-wise kernel with the same results.
 * Validation (before any CUDA call): NULL pointers, F == 0, H or W zero or odd, or F*H*W*3 bytes beyond SIZE_MAX ->
 * GFPP_ERR_INVALID.  One launch, stream-ordered, no host sync, no allocation. */
GFPP_API int gfpp_rgb_u8_to_i420(const uint8_t *rgb, uint32_t F, uint32_t H, uint32_t W, uint8_t *out, void *stream);

/* ------------------------------------------------------------------ (O) gradients of the SR head
 *
 * The SR tasks' losses (sr_mse_loss and LPIPS on sr_net(rgb_map), tasks/radnerfs/radnerf_sr.py, radnerf_torso_sr.py) need the
 * SR head's gradient w.r.t. its input image and w.r.t. its parameters.  The parameters enter as the folded matrices of
 * gfpp_sr_desc; the caller carries their gradients on to the checkpoint's parameters through the fold.
 *
 * gfpp_sr_forward_train: the four launches of gfpp_sr_forward (same out, clamp01 = 0) that also keep the activations the
 *   backward needs in `saved` (gfpp_sr_train_workspace_bytes(n_frames, in_res) bytes, 256-byte aligned); `saved` is also the
 *   forward's workspace.
 * gfpp_sr_backward: given grad_out [F, 3, 2*in_res, 2*in_res] (the gradient w.r.t. out), the same model, rgb_in and `saved` of
 *   the training forward, and the RAW noise planes (not multiplied by noise_strength; the layout of gfpp_sr_forward's, NULL
 *   entries / array: no noise term), writes
 *     grad_in [F, in_res*in_res, 3]  w.r.t. rgb_in;  NULL: skipped (the input needs no gradient)
 *     grad    w.r.t. the folded matrices, biases, toRGB weights and biases and the four noise strengths (sum over pixels and
 *             channels of the layer's pre-activation gradient times the raw plane);  NULL: no weight gradient is computed
 *   At least one of them must be given.  Gradients are fp32; the three tensor-core layers run dgrad and wgrad on TF32 wgmma with
 *   fp32 accumulation (the gradient operand rounded to nearest tf32, the other operand fp16 values of the forward).  Reductions
 *   are per-CTA partials over a fixed slicing summed in a fixed order: repeated calls are bit-identical.
 *   workspace: gfpp_sr_backward_workspace_bytes(n_frames, in_res) bytes, 256-byte aligned.
 * in_res a multiple of 128 up to 1024; no host sync, no allocation; gfpp_last_launch_count() gives the launches. */
typedef struct {
    float *conv_in_w;          /* [27][128] */
    float *conv0_w;            /* [128][1152] */
    float *up_w;               /* [256][1152] */
    float *conv1_w;            /* [64][576] */
    float *bias[4];            /* 128, 128, 64, 64 */
    float *noise_strength;     /* [4] */
    float *rgb_w[2];           /* [3][128], [3][64] */
    float *rgb_b[2];           /* [3], [3] */
} gfpp_sr_grad;

GFPP_API size_t gfpp_sr_train_workspace_bytes(uint32_t n_frames, uint32_t in_res);
GFPP_API size_t gfpp_sr_backward_workspace_bytes(uint32_t n_frames, uint32_t in_res);
GFPP_API int gfpp_sr_forward_train(const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in,
                                   const float *const noise[4], uint32_t noise_per_frame, float *out, void *saved,
                                   size_t saved_bytes, void *stream);
GFPP_API int gfpp_sr_backward(const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in, const void *saved,
                              size_t saved_bytes, const float *const noise_raw[4], uint32_t noise_per_frame, const float *grad_out,
                              float *grad_in, const gfpp_sr_grad *grad, void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* GFPP_H_ */
