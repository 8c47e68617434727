// capi.cu -- extern "C" boundary of libgfpp.so (see include/gfpp.h for the contract).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "../../include/gfpp.h"
#include "common.cuh"
#include "field_train_kernel.cuh"
#include "field_train_tc_kernel.cuh"
#include "grid_half.cuh"
#include "head_kernel.cuh"
#include "launch.cuh"
#include "sr_kernel.cuh"
#include "torso_grid_kernel.cuh"
#include "torso_kernel.cuh"
#include "torso_sr_kernel.cuh"
#include "torso_train_kernel.cuh"

namespace gfpp {
// ops_kernels.cu
cudaError_t launch_near_far(const float *, const float *, const float *, uint32_t, float, float *, float *, cudaStream_t);
cudaError_t launch_march_rays(const MarchConst &, uint32_t, uint32_t, const int32_t *, const float *, const float *,
                              const float *, const float *, float *, float *, float *, const float *, cudaStream_t);
cudaError_t launch_composite_rays(uint32_t, uint32_t, float, int32_t *, float *, const float *, const float *,
                                  const float *, float *, float *, float *, cudaStream_t);
cudaError_t launch_grid_encode(const GridMeta &, const float *, const float *, float *, uint32_t, cudaStream_t);
cudaError_t launch_sh_encode(const float *, float *, uint32_t, uint32_t, cudaStream_t);
cudaError_t launch_freq_encode(const float *, uint32_t, uint32_t, uint32_t, float *, cudaStream_t);
cudaError_t launch_occupancy_bounds(const uint8_t *, uint32_t, uint32_t, int *, cudaStream_t);
cudaError_t launch_coarse_occupancy(const uint8_t *, uint32_t, uint32_t, uint32_t *, cudaStream_t);
cudaError_t launch_pack_quads(const GridMeta &, const float *, float *, uint32_t, cudaStream_t);
cudaError_t launch_pack_octs(const GridMeta &, const float *, void *, uint32_t, cudaStream_t);
cudaError_t launch_pack_octs_i16(const GridMeta &, const float *, void *, uint32_t, uint32_t *, float *, cudaStream_t);
// tc_pack.cu
cudaError_t launch_pack_tc_tile(const float *, int, int, int, int, int, int, int, int, unsigned char *, unsigned char *, cudaStream_t);
cudaError_t launch_pack_fold_tile(const float *, int, int, const float *, unsigned char *, int, cudaStream_t);
cudaError_t launch_tc_selftest(const float *, int, const unsigned char *, const unsigned char *, int, int, int, int, float *, cudaStream_t);
// train_kernels.cu
size_t march_train_scratch_bytes(uint32_t N);
cudaError_t launch_march_rays_train(const MarchConst &, const float *, const float *, const float *, const float *, const float *, uint32_t,
                                    uint32_t, uint32_t, float *, float *, float *, int *, int *, int *, int *, cudaStream_t);
cudaError_t launch_march_rays_train_backward(const float *, const float *, const int *, const float *, uint32_t, uint32_t, float *, float *,
                                             cudaStream_t);
cudaError_t launch_composite_train_forward(const float *, const float *, const float *, const float *, const int *, uint32_t, uint32_t, float,
                                           float *, float *, float *, float *, cudaStream_t);
cudaError_t launch_composite_train_backward(const float *, const float *, const float *, const float *, const float *, const float *,
                                            const float *, const int *, const float *, const float *, const float *, uint32_t, uint32_t, float,
                                            float *, float *, float *, cudaStream_t);
cudaError_t launch_grid_encode_dydx(const GridMeta &, const float *, const float *, float *, float *, uint32_t, cudaStream_t);
cudaError_t launch_grid_backward(const GridMeta &, const float *, const float *, float *, const float *, float *, uint32_t, int *, cudaStream_t);
cudaError_t launch_grad_tv(const GridMeta &, const float *, const float *, float *, float, uint32_t, cudaStream_t);
cudaError_t launch_packbits(const float *, uint32_t, float, uint8_t *, cudaStream_t);
cudaError_t launch_morton3D(const int *, uint32_t, int *, cudaStream_t);
cudaError_t launch_morton3D_invert(const int *, uint32_t, int *, cudaStream_t);
cudaError_t launch_morton3D_dilation(const float *, uint32_t, uint32_t, float *, cudaStream_t);
cudaError_t launch_sph_from_ray(const float *, const float *, float, uint32_t, float *, cudaStream_t);
// grid_kernels.cu
uint32_t dilate_ema_blocks(uint32_t C, uint32_t H);
cudaError_t launch_grid_refresh_tail(const float *, uint32_t, uint32_t, float, float, float *, double *, float *, float *, uint8_t *, int *,
                                     cudaStream_t);
cudaError_t launch_mark_untrained(const float *, uint32_t, float, float, const float *, const float *, uint32_t, uint32_t, float *, cudaStream_t);
uint32_t torso_dilate_ema_blocks(uint32_t H);
cudaError_t launch_torso_grid_tail(const float *, uint32_t, float, float, float *, double *, float *, float *, int *, cudaStream_t);
// torso_pass_kernels.cu
uint32_t torso_mask_tiles(uint32_t N);
cudaError_t launch_torso_mask(const float *, uint32_t, float, const float *, const float *, const float *, uint32_t, int32_t *, int32_t *,
                              float *, float *, float *, int32_t *, int *, cudaStream_t);
cudaError_t launch_torso_composite_fwd(const int32_t *, uint32_t, const float *, const float *, const float *, const float *, const float *,
                                       uint32_t, float *, float *, float *, cudaStream_t);
cudaError_t launch_torso_composite_bwd(const int32_t *, uint32_t, const float *, const float *, const float *, const float *, const float *,
                                       uint32_t, const float *, const float *, const float *, float *, float *, cudaStream_t);
}  // namespace gfpp

using namespace gfpp;

namespace {

// per-thread state only (the library is thread-compatible: nothing below is shared between host threads)
thread_local char g_err[512] = "";
thread_local int g_launches = 0;
thread_local bool g_profile = false;                 // opt-in diagnostics of the calling thread (bench.py, tools/phase_breakdown.py)
thread_local unsigned long long *g_phase = nullptr;
thread_local cudaEvent_t g_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
thread_local int g_ev_dev = -1;                      // device the events were created on

int fail(int code, const char *fmt, const char *detail = "") {
    snprintf(g_err, sizeof(g_err), fmt, detail);
    return code;
}

// CK: a kernel launch (counted in gfpp_last_launch_count); CKN: any other runtime call
#define CK(expr)                                                                      \
    do {                                                                              \
        cudaError_t e__ = (expr);                                                     \
        if (e__ != cudaSuccess) return fail(GFPP_ERR_CUDA, #expr ": %s", cudaGetErrorString(e__)); \
        ++g_launches;                                                                 \
    } while (0)
#define CKN(expr)                                                                     \
    do {                                                                              \
        cudaError_t e__ = (expr);                                                     \
        if (e__ != cudaSuccess) return fail(GFPP_ERR_CUDA, #expr ": %s", cudaGetErrorString(e__)); \
    } while (0)

// Level constants exactly as the reference kernel derives them (gridencoder.cu:137-139, :66-84), computed once on
// the host with the same libm calls as oracle/native_ops.c.
int fill_grid_meta(GridMeta &gm, const int32_t *offsets, uint32_t D, uint32_t L, float S, uint32_t H,
                   uint32_t gridtype, int align_corners, uint32_t interp) {
    if (L == 0 || L > GFPP_MAX_LEVELS || (D != 2 && D != 3) || !offsets) return -1;
    memset(&gm, 0, sizeof(gm));
    gm.num_levels = L;
    gm.dim = D;
    gm.interp = interp;
    gm.align_off = align_corners ? 0.0f : 0.5f;
    bool quad_ok = true;
    for (uint32_t l = 0; l < L; ++l) {
        const float scale = exp2f((float)l * S) * (float)H - 1.0f;
        const uint32_t res = (uint32_t)ceil((double)scale) + 1;
        const uint32_t hs = (uint32_t)(offsets[l + 1] - offsets[l]);
        const uint32_t step = align_corners ? res : res + 1;
        gm.scale[l] = scale;
        gm.offset[l] = (uint32_t)offsets[l];
        gm.hsize[l] = hs;
        gm.hmask[l] = (hs & (hs - 1)) == 0 ? hs - 1 : 0;
        uint32_t stride = 1;
        uint32_t mul[3] = {0, 0, 0};
        for (uint32_t d = 0; d < D && stride <= hs; ++d) {
            mul[d] = stride;
            stride *= step;  // uint32 wrap on purpose, as in the reference
        }
        if (mul[0] != 1) return -1;  // hashmap_size 0
        gm.mul1[l] = mul[1];
        gm.mul2[l] = mul[2];
        gm.hashed[l] = (gridtype == 0 && stride > hs) ? 1u : 0u;
        // the packed-corner layout needs corner slots = base + const offsets, consistently under the level's modulo
        const unsigned long long span = (unsigned long long)(res + 1) * (1ull + mul[1] + mul[2]);
        if (gm.hashed[l] || (gm.hmask[l] == 0 && span >= (1ull << 32))) quad_ok = false;
    }
    gm.quad_ok = quad_ok ? 1u : 0u;
    return 0;
}

// ---------------------------------------------------------------- packed model
constexpr int kChunkK[HEAD_NCHUNK] = {48, 48, 64, 64, 64, 64, 64, 64, 64, 72, 72};

struct ModelHost {
    uint32_t magic;
    int has_torso;
    GridMeta pos_gm, amb_gm, tor_gm;
    const float2 *pos_tab, *amb_tab, *tor_tab;
    const float4 *pos_quads, *amb_quads;
    const uint4 *pos_octs, *amb_octs;
    const uint8_t *bitfield;
    const float *density_grid_torso;
    const float *torso_def0_src, *torso_can0_src, *torso_code;  // originals (per-frame bias fold reads them)
    uint32_t torso_code_dim;
    // into packed
    const float *wide, *narrow;
    const float *wd0, *wd1, *wd2, *wc0, *wc1, *wc2;
    const int *occ_bounds;
    const uint32_t *coarse_bits;
    int coarse_words;
    int chunk_off[HEAD_NCHUNK];
    float aabb[6];
    float bound, min_near, density_scale, density_thresh_torso, torso_shrink;
    uint32_t cascade, grid_size;
    int use_occ_box;
    int mlp_precision;
    HeadTcArgs tc;
    // v2 head kernel (head_v2_kernel.cu): shared weight stream + resident tiles; valid when v2_ok
    int v2_ok;
    const unsigned char *v2_stream, *v2_res;
    const float *v2_pos_step;       // robust mode: per-level step of the 16-bit position table
    const float *amb0_src;          // ambient_net.net.0.weight [128,96] (its conditioning columns are folded per frame)
    const float *color0_src;        // color_net.net.0.weight [128, 144 + ind_dim] (gfpp_frozen_head folds a per-call code into a copy of `narrow`)
    int ind_dim;
    const unsigned char *tor_tf32;  // tf32 hi / lo images of the wide torso layers (k_epilogue)
};
static_assert(sizeof(ModelHost) <= sizeof(gfpp_model), "gfpp_model opaque storage too small");
constexpr uint32_t kMagic = 0x67667070u;  // "gfpp"

struct PackedLayout {
    size_t wide, narrow, wd0, wd1, wd2, wc0, wc1, wc2, tor_tf32, occ, coarse, tc_hi, tc_lo, v2_stream, v2_res, v2_step, pos_quads, amb_quads, total;
};

// tensor-core weight stream: kHeadTcChunks (head_kernel.cuh)
using TcChunk = HeadTcChunk;
constexpr const HeadTcChunk *kTc = kHeadTcChunks;
inline int tc_chunk_bytes(int c) { return kTc[c].rows * (kTc[c].k16 ? 32 : 128); }

inline size_t coarse_words_for(uint32_t cascade, uint32_t grid_size) {
    const size_t hc = grid_size / 4;
    return (cascade * hc * hc * hc + 31) / 32;
}

PackedLayout packed_layout(uint32_t cascade = 8, uint32_t grid_size = 128, size_t pos_entries = 0, size_t amb_entries = 0) {
    PackedLayout L;
    size_t o = 0;
    auto take = [&](size_t floats) { size_t r = o; o += (floats * 4 + 255) / 256 * 256; return r; };
    size_t wide = 0;
    for (int c = 0; c < HEAD_NCHUNK; ++c) wide += (size_t)kChunkK[c] * 128;
    L.wide = take(wide);
    L.narrow = take(8 * 128);
    L.wd0 = take(44 * 64);
    L.wd1 = take(64 * 64);
    L.wd2 = take(2 * 64);
    L.wc0 = take(76 * 32);
    L.wc1 = take(32 * 32);
    L.wc2 = take(4 * 32);
    L.tor_tf32 = take(TORSO_TF32_BYTES / 4);
    L.occ = take(8);
    L.coarse = take(coarse_words_for(cascade, grid_size));
    size_t tcb = 0;
    for (int c = 0; c < HEAD_TC_NCHUNK; ++c) tcb += (size_t)tc_chunk_bytes(c);
    L.tc_hi = take(tcb / 4);
    L.tc_lo = take(tcb / 4);
    L.v2_stream = take((size_t)V2_NTILE_ROBUST * V2_TILE_BYTES / 4);
    L.v2_res = take(V2_RES_BYTES / 4);
    L.v2_step = take(64);          // 16 steps + 16 words of scratch for the per-level maxima
    L.pos_quads = take(pos_entries * 8);   // 32 bytes per entry
    L.amb_quads = take(amb_entries * 8);
    L.total = o;
    return L;
}

struct WorkLayout {
    size_t image, rays_t, wsum, depth, survivors, hits, zero_begin, hist, counters, B_total, valid, pcount, zero_end, bias_def,
        bias_can, bias_amb, total;
};

WorkLayout work_layout(uint32_t F, uint32_t N, uint32_t max_steps) {
    WorkLayout W;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    const size_t FN = (size_t)F * N;
    W.image = take(FN * 3 * 4);
    W.rays_t = take(FN * 4);
    W.wsum = take(FN * 4);
    W.depth = take(FN * 4);
    W.survivors = take(FN * 4);
    W.hits = take(FN * 64);   // HitRecord (head_common.cuh)
    W.zero_begin = o;
    W.hist = take((size_t)F * (max_steps + 2) * 4);
    W.counters = take(16 * 4);
    W.B_total = take((size_t)F * 4);
    W.valid = take((size_t)F * 4);
    W.pcount = take((size_t)F * 4);
    W.zero_end = o;
    W.bias_def = take((size_t)F * 64 * 4);
    W.bias_can = take((size_t)F * 32 * 4);
    W.bias_amb = take((size_t)F * 64 * 2 * 2);   // fp16 hi + lo images of the conditioning vectors (v2 head kernel)
    W.total = o;
    return W;
}

__global__ void k_init_bounds(int *b) {
    if (threadIdx.x < 3) b[threadIdx.x] = INT_MAX;
    else if (threadIdx.x < 6) b[threadIdx.x] = -1;
}

__global__ void k_write_stats(const int *B_total, const int *n_survivors, const int *valid, const int *pcount, int F,
                              int32_t *stats) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    stats[4 * f] = B_total[f];
    stats[4 * f + 1] = *n_survivors;
    stats[4 * f + 2] = valid[f];
    stats[4 * f + 3] = pcount[f];
}

}  // namespace

extern "C" {

const char *gfpp_last_error(void) { return g_err; }
int gfpp_version(void) { return 100; }
int gfpp_last_launch_count(void) { return g_launches; }

int gfpp_profile_enable(int on) {
    int dev = -1;
    if (on && cudaGetDevice(&dev) != cudaSuccess) return fail(GFPP_ERR_CUDA, "no CUDA device%s");
    if (on && (!g_ev[0] || g_ev_dev != dev)) {   // events belong to a device: (re)create them for the current one
        for (int i = 0; i < 5; ++i) {
            if (g_ev[i]) cudaEventDestroy(g_ev[i]);
            if (cudaEventCreate(&g_ev[i]) != cudaSuccess) return fail(GFPP_ERR_CUDA, "cudaEventCreate failed%s");
        }
        g_ev_dev = dev;
    }
    g_profile = on != 0;
    return GFPP_OK;
}

int gfpp_profile_phases(void *dev_u64x32) {
    g_phase = (unsigned long long *)dev_u64x32;
    return GFPP_OK;
}

int gfpp_profile_read(float ms[4]) {
    if (!g_profile || !g_ev[0] || !ms) return fail(GFPP_ERR_INVALID, "profile_read: profiling is not enabled%s");
    CKN(cudaEventSynchronize(g_ev[3]));
    for (int i = 0; i < 3; ++i) CKN(cudaEventElapsedTime(&ms[i], g_ev[i], g_ev[i + 1]));
    CKN(cudaEventElapsedTime(&ms[3], g_ev[4], g_ev[0]));   // everything before the head kernel: memset, torso biases, ray setup
    return GFPP_OK;
}

int gfpp_check_device(void) {
    int dev = 0;
    cudaDeviceProp p;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&p, dev) != cudaSuccess)
        return fail(GFPP_ERR_CUDA, "no CUDA device%s");
    if (p.major != 9 || p.minor != 0) {
        snprintf(g_err, sizeof(g_err), "libgfpp is built for sm_90a only; device is sm_%d%d", p.major, p.minor);
        return GFPP_ERR_UNSUPPORTED;
    }
    return GFPP_OK;
}

// ------------------------------------------------------------------ (A) per-op mirror
int gfpp_near_far_from_aabb(const float *rays_o, const float *rays_d, const float *aabb, uint32_t N, float min_near,
                            float *nears, float *fars, void *stream) {
    if (!rays_o || !rays_d || !aabb || !nears || !fars) return fail(GFPP_ERR_INVALID, "near_far_from_aabb: null pointer%s");
    g_launches = 0;
    CK(launch_near_far(rays_o, rays_d, aabb, N, min_near, nears, fars, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t *rays_alive, const float *rays_t,
                    const float *rays_o, const float *rays_d, float bound, float dt_gamma, uint32_t max_steps, uint32_t C,
                    uint32_t H, const uint8_t *grid, const float *nears, const float *fars, float *xyzs, float *dirs,
                    float *deltas, const float *noises, void *stream) {
    (void)nears;
    if (!rays_alive || !rays_t || !rays_o || !rays_d || !grid || !fars || !xyzs || !dirs || !deltas || !noises)
        return fail(GFPP_ERR_INVALID, "march_rays: null pointer%s");
    if (C < 1 || C > 8 || H < 1 || H > 1024 || max_steps < 1) return fail(GFPP_ERR_INVALID, "march_rays: bad C/H/max_steps%s");
    MarchConst mc;
    march_const_init(mc, bound, dt_gamma, max_steps, C, H, grid);
    g_launches = 0;
    CK(launch_march_rays(mc, n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, fars, xyzs, dirs, deltas, noises,
                         (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t *rays_alive, float *rays_t,
                        const float *sigmas, const float *rgbs, const float *deltas, float *weights_sum, float *depth,
                        float *image, void *stream) {
    if (!rays_alive || !rays_t || !sigmas || !rgbs || !deltas || !weights_sum || !depth || !image)
        return fail(GFPP_ERR_INVALID, "composite_rays: null pointer%s");
    g_launches = 0;
    CK(launch_composite_rays(n_alive, n_step, T_thresh, rays_alive, rays_t, sigmas, rgbs, deltas, weights_sum, depth,
                             image, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_grid_encode_forward(const float *inputs, const float *embeddings, const int32_t *offsets_host, float *outputs,
                             uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, uint32_t gridtype,
                             int align_corners, uint32_t interp, void *stream) {
    if (!inputs || !embeddings || !offsets_host || !outputs) return fail(GFPP_ERR_INVALID, "grid_encode_forward: null pointer%s");
    // the reference throws std::runtime_error for unsupported C / D (gridencoder.cu:380, 397)
    if (C != 2) return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: this build supports C == 2 only%s");
    GridMeta gm;
    if (fill_grid_meta(gm, offsets_host, D, L, S, H, gridtype, align_corners, interp) != 0)
        return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: D must be 2 or 3 and L <= 16%s");
    g_launches = 0;
    CK(launch_grid_encode(gm, inputs, embeddings, outputs, B, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_sh_encode_forward(const float *inputs, float *outputs, uint32_t B, uint32_t D, uint32_t degree, void *stream) {
    if (!inputs || !outputs) return fail(GFPP_ERR_INVALID, "sh_encode_forward: null pointer%s");
    if (D != 3 || degree < 1 || degree > 4) return fail(GFPP_ERR_UNSUPPORTED, "SH encoder: D must be 3 and degree in 1..4%s");
    g_launches = 0;
    CK(launch_sh_encode(inputs, outputs, B, degree, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_freq_encode_forward(const float *inputs, uint32_t B, uint32_t D, uint32_t deg, uint32_t C, float *outputs,
                             void *stream) {
    if (!inputs || !outputs) return fail(GFPP_ERR_INVALID, "freq_encode_forward: null pointer%s");
    if (C != D + 2 * D * deg) return fail(GFPP_ERR_INVALID, "freq_encode_forward: C != D + 2*D*deg%s");
    g_launches = 0;
    CK(launch_freq_encode(inputs, B, D, C, outputs, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_tc_selftest(const float *A, const float *W, uint32_t N, uint32_t K, int k16_tail, int precision, void *scratch,
                     float *out, void *stream) {
    if (!A || !W || !scratch || !out) return fail(GFPP_ERR_INVALID, "tc_selftest: null pointer%s");
    const int k64 = (int)K - (k16_tail ? 16 : 0);
    if ((N != 16 && N != 128 && N != 144) || k64 <= 0 || k64 % 16 || K > 144 || precision < 1 || precision > 3)
        return fail(GFPP_ERR_INVALID, "tc_selftest: unsupported shape%s");
    const int nt64 = (k64 + 63) / 64;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char *hi = (unsigned char *)scratch, *lo = hi + 3 * 18432;
    const int bf16 = precision != 1;
    g_launches = 0;
    CKN(cudaMemsetAsync(scratch, 0, 6 * 18432, st));
    for (int t = 0; t < nt64; ++t) {
        const int kc = (k64 - t * 64) < 64 ? (k64 - t * 64) : 64;
        CK(launch_pack_tc_tile(W, (int)K, 0, t * 64, (int)N, kc, 0, 0, bf16, hi + t * 18432, precision == 2 ? lo + t * 18432 : nullptr, st));
    }
    if (k16_tail)
        CK(launch_pack_tc_tile(W, (int)K, 0, k64, (int)N, 16, 0, 1, bf16, hi + nt64 * 18432, precision == 2 ? lo + nt64 * 18432 : nullptr, st));
    CK(launch_tc_selftest(A, (int)K, hi, lo, (int)N, nt64, k16_tail, precision, out, st));
    return GFPP_OK;
}

// ------------------------------------------------------------------ (B) fused renderer
size_t gfpp_model_packed_bytes(const gfpp_model_desc *desc) {
    if (!desc) return packed_layout().total;
    const gfpp_grid_desc &p = desc->position_grid, &q = desc->ambient_grid;
    const size_t pe = p.offsets_host && p.num_levels <= 16 ? (size_t)p.offsets_host[p.num_levels] : 0;
    const size_t ae = q.offsets_host && q.num_levels <= 16 ? (size_t)q.offsets_host[q.num_levels] : 0;
    return packed_layout(desc->cascade, desc->grid_size, pe, ae).total;
}

int gfpp_model_pack(const gfpp_model_desc *d, void *packed, size_t packed_bytes, gfpp_model *model, void *stream) {
    if (!d || !packed || !model) return fail(GFPP_ERR_INVALID, "model_pack: null pointer%s");
    if (d->cascade < 1 || d->cascade > 8 || d->grid_size < 8 || d->grid_size > 1024 || d->grid_size % 4)
        return fail(GFPP_ERR_UNSUPPORTED, "model_pack: cascade/grid_size out of range%s");
    if (!d->position_grid.offsets_host || !d->ambient_grid.offsets_host || d->position_grid.num_levels > 16 || d->ambient_grid.num_levels > 16)
        return fail(GFPP_ERR_INVALID, "model_pack: grid offsets missing%s");
    const size_t pos_entries = (size_t)d->position_grid.offsets_host[d->position_grid.num_levels];
    const size_t amb_entries = (size_t)d->ambient_grid.offsets_host[d->ambient_grid.num_levels];
    const PackedLayout L = packed_layout(d->cascade, d->grid_size, pos_entries, amb_entries);
    if (packed_bytes < L.total) return fail(GFPP_ERR_WORKSPACE, "model_pack: packed buffer too small%s");
    if (d->cond_dim != 64 || d->ind_dim > 16) return fail(GFPP_ERR_UNSUPPORTED, "model_pack: cond_dim must be 64, ind_dim <= 16%s");
    if (d->cascade < 1 || d->cascade > 8 || d->grid_size < 8 || d->grid_size > 1024)
        return fail(GFPP_ERR_UNSUPPORTED, "model_pack: cascade/grid_size out of range%s");
    for (int i = 0; i < 3; ++i)
        if (!d->ambient_w[i] || !d->sigma_w[i]) return fail(GFPP_ERR_INVALID, "model_pack: null weight%s");
    if (!d->color_w[0] || !d->color_w[1] || !d->density_bitfield) return fail(GFPP_ERR_INVALID, "model_pack: null weight%s");
    cudaStream_t st = (cudaStream_t)stream;
    ModelHost m;
    memset(&m, 0, sizeof(m));
    m.magic = kMagic;
    const gfpp_grid_desc *gd[3] = {&d->position_grid, &d->ambient_grid, &d->torso_grid};
    GridMeta *gm[3] = {&m.pos_gm, &m.amb_gm, &m.tor_gm};
    for (int i = 0; i < (d->has_torso ? 3 : 2); ++i) {
        if (!gd[i]->embeddings) return fail(GFPP_ERR_INVALID, "model_pack: null grid table%s");
        if (gd[i]->num_levels != 16)
            return fail(GFPP_ERR_UNSUPPORTED, "model_pack: grids must have 16 levels x 2 features%s");
        if (fill_grid_meta(*gm[i], gd[i]->offsets_host, gd[i]->input_dim, gd[i]->num_levels, gd[i]->log2_per_level_scale,
                           gd[i]->base_resolution, gd[i]->gridtype, gd[i]->align_corners, gd[i]->interp) != 0)
            return fail(GFPP_ERR_UNSUPPORTED, "model_pack: unsupported grid layout%s");
    }
    if (m.pos_gm.dim != 3) return fail(GFPP_ERR_UNSUPPORTED, "model_pack: position grid must be 3-D%s");
    if (d->has_torso && m.tor_gm.dim != 2) return fail(GFPP_ERR_UNSUPPORTED, "model_pack: torso grid must be 2-D%s");
    m.pos_tab = (const float2 *)d->position_grid.embeddings;
    m.amb_tab = (const float2 *)d->ambient_grid.embeddings;
    m.tor_tab = d->has_torso ? (const float2 *)d->torso_grid.embeddings : nullptr;
    m.bitfield = d->density_bitfield;
    memcpy(m.aabb, d->aabb, sizeof(m.aabb));
    m.bound = d->bound;
    m.min_near = d->min_near;
    m.density_scale = d->density_scale;
    m.cascade = d->cascade;
    m.grid_size = d->grid_size;
    const float cube = d->bound;
    m.use_occ_box = (d->cascade == 1 && d->aabb[0] >= -cube && d->aabb[1] >= -cube && d->aabb[2] >= -cube &&
                     d->aabb[3] <= cube && d->aabb[4] <= cube && d->aabb[5] <= cube) ? 1 : 0;

    char *base = (char *)packed;
    float *wide = (float *)(base + L.wide), *narrow = (float *)(base + L.narrow);
    g_launches = 0;
    // stream order of the wide chunks (k-rows of the transposed weights): ambient L0 (96 = 48+48), ambient L1 (64+64),
    // sigma L0 (64), sigma L1 (64+64), sigma L2 geo rows 1..128 (64+64), color L0 columns 0..143 (72+72)
    struct Src { const float *w; int ld, row0, col0; };
    const int amb_dim = (int)m.amb_gm.dim;
    const int col0_in = 16 + 128 + (int)d->ind_dim;
    const Src src[HEAD_NCHUNK] = {
        {d->ambient_w[0], 96, 0, 0},  {d->ambient_w[0], 96, 0, 48}, {d->ambient_w[1], 128, 0, 0}, {d->ambient_w[1], 128, 0, 64},
        {d->sigma_w[0], 64, 0, 0},    {d->sigma_w[1], 128, 0, 0},   {d->sigma_w[1], 128, 0, 64},  {d->sigma_w[2], 128, 1, 0},
        {d->sigma_w[2], 128, 1, 64},  {d->color_w[0], col0_in, 0, 0}, {d->color_w[0], col0_in, 0, 72}};
    int off = 0;
    for (int c = 0; c < HEAD_NCHUNK; ++c) {
        m.chunk_off[c] = off;
        CK(launch_pack_kmajor(src[c].w, src[c].ld, src[c].row0, src[c].col0, 128, kChunkK[c], kChunkK[c], wide + off, st));
        off += kChunkK[c] * 128;
    }
    CKN(cudaMemsetAsync(narrow, 0, 8 * 128 * 4, st));
    CK(launch_pack_rows(d->ambient_w[2], 128, 0, amb_dim, 128, 128, narrow, st));            // rows 0..2
    CK(launch_pack_rows(d->sigma_w[2], 128, 0, 1, 128, 128, narrow + 3 * 128, st));           // row 3: sigma
    CK(launch_pack_rows(d->color_w[1], 128, 0, 3, 128, 128, narrow + 4 * 128, st));           // rows 4..6
    if (d->ind_dim > 0)
        CK(launch_fold_bias(d->color_w[0], col0_in, 144, (int)d->ind_dim, d->individual_code, 128, narrow + 7 * 128, st));
    m.wide = wide;
    m.narrow = narrow;

    int *occ = (int *)(base + L.occ);
    k_init_bounds<<<1, 32, 0, st>>>(occ);
    CK(cudaGetLastError());
    const uint32_t H3 = d->grid_size * d->grid_size * d->grid_size;
    CK(launch_occupancy_bounds(d->density_bitfield, d->cascade * H3 / 8, H3, occ, st));
    m.occ_bounds = occ;
    // coarse (4x4x4 OR-pooled) occupancy: lets the marcher skip empty space without touching the fine bitfield
    uint32_t *coarse = (uint32_t *)(base + L.coarse);
    m.coarse_words = (int)coarse_words_for(d->cascade, d->grid_size);
    CKN(cudaMemsetAsync(coarse, 0, (size_t)m.coarse_words * 4, st));
    CK(launch_coarse_occupancy(d->density_bitfield, d->cascade, d->grid_size, coarse, st));
    m.coarse_bits = coarse;

    // sector-packed corner copies of the two head grids (tiled layouts only); done before the tensor-core weight
    // packing below because that one clears everything from tc_hi to the END of the packed buffer
    const bool want_quads = getenv("GFPP_NO_QUADS") == nullptr;
    m.mlp_precision = (int)d->mlp_precision;
    if (d->mlp_precision > 4) return fail(GFPP_ERR_UNSUPPORTED, "model_pack: mlp_precision must be 0..4%s");
    const bool robust = d->mlp_precision == 4;
    if (d->mlp_precision != 0) CKN(cudaMemsetAsync(base + L.tc_hi, 0, L.pos_quads - L.tc_hi, st));
    m.amb0_src = d->ambient_w[0];
    m.color0_src = d->color_w[0];
    m.ind_dim = (int)d->ind_dim;
    if (d->mlp_precision == 1 || robust) {
        // v2 weight images: streamed tiles in the kernel's schedule order (head_kernel.cuh), then the resident block
        unsigned char *vs = (unsigned char *)(base + L.v2_stream), *vr = (unsigned char *)(base + L.v2_res);
        struct T { const float *w; int ld, row0, col0, kc; bool split; };
        const T tiles[7] = {{d->ambient_w[0], 96, 0, 0, 64, true},  {d->ambient_w[0], 96, 0, 64, 32, true},
                            {d->ambient_w[1], 128, 0, 0, 64, true}, {d->ambient_w[1], 128, 0, 64, 64, true},
                            {d->sigma_w[0], 64, 0, 0, 64, false},   {d->sigma_w[1], 128, 0, 0, 64, false},  {d->sigma_w[1], 128, 0, 64, 64, false}};
        int ti = 0;
        for (int c = 0; c < 7; ++c) {
            const bool sp = robust && tiles[c].split;
            unsigned char *hi = vs + (size_t)ti * V2_TILE_BYTES, *lo = sp ? hi + V2_TILE_BYTES : nullptr;
            CK(launch_pack_tc_tile(tiles[c].w, tiles[c].ld, tiles[c].row0, tiles[c].col0, 128, tiles[c].kc, 0, 0, 0, hi, lo, st));
            ti += sp ? 2 : 1;
        }
        // the last two: sigma L2's geo rows folded into color L0's geo columns (one fp16 image in both modes, DESIGN §6)
        CK(launch_pack_fold_tile(d->color_w[0], col0_in, 16, d->sigma_w[2], vs + (size_t)ti * V2_TILE_BYTES, V2_TILE_BYTES, st));
        static_assert(V2_NTILE_X1 == 7 + 2 && V2_NTILE_ROBUST == 7 + 4 + 2, "v2 tile table");
        for (int kt = 0; kt < 2; ++kt) {
            CK(launch_pack_tc_tile(d->ambient_w[2], 128, 0, kt * 64, amb_dim, 64, 0, 0, 0, vr + V2_RES_AMBN_HI + kt * 2048,
                                   robust ? vr + V2_RES_AMBN_LO + kt * 2048 : nullptr, st));
            CK(launch_pack_tc_tile(d->sigma_w[2], 128, 0, kt * 64, 1, 64, 0, 0, 0, vr + V2_RES_SIGROW + kt * 2048, nullptr, st));
            CK(launch_pack_tc_tile(d->color_w[1], 128, 0, kt * 64, 3, 64, 0, 0, 0, vr + V2_RES_COLN + kt * 2048, nullptr, st));
        }
        CK(launch_pack_tc_tile(d->color_w[0], col0_in, 0, 0, 128, 16, 0, 1, 0, vr + V2_RES_COLSH, nullptr, st));
        m.v2_stream = vs; m.v2_res = vr;
    }
    if (d->mlp_precision != 0 && !robust) {
        const int bf16 = d->mlp_precision != 1;
        const bool split = d->mlp_precision == 2;
        unsigned char *thi = (unsigned char *)(base + L.tc_hi), *tlo = (unsigned char *)(base + L.tc_lo);
        const float *lw[6] = {d->ambient_w[0], d->ambient_w[1], d->sigma_w[0], d->sigma_w[1], d->sigma_w[2], d->color_w[0]};
        const int lld[6] = {96, 128, 64, 128, 128, col0_in};
        int boff = 0;
        for (int c = 0; c < HEAD_TC_NCHUNK; ++c) {
            const TcChunk &k = kTc[c];
            if (k.layer == 4) {  // sigma L2: geo rows (W rows 1..128) first, the sigma row (W row 0) as row 128
                CK(launch_pack_tc_tile(lw[4], 128, 1, k.col0, 128, k.kc, 0, 0, bf16, thi + boff, split ? tlo + boff : nullptr, st));
                CK(launch_pack_tc_tile(lw[4], 128, 0, k.col0, 1, k.kc, 128, 0, bf16, thi + boff, split ? tlo + boff : nullptr, st));
            } else {
                CK(launch_pack_tc_tile(lw[k.layer], lld[k.layer], 0, k.col0, 128, k.kc, 0, k.k16, bf16, thi + boff, split ? tlo + boff : nullptr, st));
            }
            boff += tc_chunk_bytes(c);
        }
        m.tc.w_hi = thi; m.tc.w_lo = tlo;
    }

    // fp16 mode: fp16 "octs" (one 32-byte sector per sample-level; tables rounded to fp16 like the reference under
    // autocast); every other mode: fp32 "quads" (bit-identical values).  Both occupy the same 32 bytes per entry.
    const bool want_octs = want_quads && (d->mlp_precision == 1 || robust) && getenv("GFPP_NO_OCTS") == nullptr;
    if (want_quads && m.pos_gm.quad_ok && m.pos_gm.dim == 3) {
        if (want_octs && robust) {   // 16-bit fixed point, one step per level: the position table's rounding is what the ambient net amplifies
            float *step = (float *)(base + L.v2_step);
            CK(launch_pack_octs_i16(m.pos_gm, d->position_grid.embeddings, base + L.pos_quads, (uint32_t)pos_entries, (uint32_t *)(step + 16), step, st));
            m.pos_octs = (const uint4 *)(base + L.pos_quads);
            m.v2_pos_step = step;
        } else if (want_octs) {
            CK(launch_pack_octs(m.pos_gm, d->position_grid.embeddings, base + L.pos_quads, (uint32_t)pos_entries, st));
            m.pos_octs = (const uint4 *)(base + L.pos_quads);
        } else {
            CK(launch_pack_quads(m.pos_gm, d->position_grid.embeddings, (float *)(base + L.pos_quads), (uint32_t)pos_entries, st));
            m.pos_quads = (const float4 *)(base + L.pos_quads);
        }
    }
    if (want_quads && m.amb_gm.quad_ok && m.amb_gm.dim == 3) {
        if (want_octs) {
            CK(launch_pack_octs(m.amb_gm, d->ambient_grid.embeddings, base + L.amb_quads, (uint32_t)amb_entries, st));
            m.amb_octs = (const uint4 *)(base + L.amb_quads);
        } else {
            CK(launch_pack_quads(m.amb_gm, d->ambient_grid.embeddings, (float *)(base + L.amb_quads), (uint32_t)amb_entries, st));
            m.amb_quads = (const float4 *)(base + L.amb_quads);
        }
    }

    m.v2_ok = (m.v2_stream && m.pos_octs && m.amb_octs && m.pos_gm.num_levels == 16 && m.amb_gm.num_levels == 16 && amb_dim == 3) ? 1 : 0;
    if (robust && !m.v2_ok)
        return fail(GFPP_ERR_UNSUPPORTED, "model_pack: the robust mode needs 3-D tiled position and ambient grids (sector-packed tables)%s");
    m.has_torso = d->has_torso;
    if (d->has_torso) {
        for (int i = 0; i < 3; ++i)
            if (!d->torso_deform_w[i] || !d->torso_canon_w[i]) return fail(GFPP_ERR_INVALID, "model_pack: null torso weight%s");
        if (!d->density_grid_torso) return fail(GFPP_ERR_INVALID, "model_pack: null density_grid_torso%s");
        if (d->torso_code_dim > 10) return fail(GFPP_ERR_UNSUPPORTED, "model_pack: torso_code_dim <= 10%s");
        const int din = 42 + 54 + (int)d->torso_code_dim;
        float *wd0 = (float *)(base + L.wd0), *wd1 = (float *)(base + L.wd1), *wd2 = (float *)(base + L.wd2);
        float *wc0 = (float *)(base + L.wc0), *wc1 = (float *)(base + L.wc1), *wc2 = (float *)(base + L.wc2);
        CK(launch_pack_kmajor(d->torso_deform_w[0], din, 0, 0, 64, 42, 44, wd0, st));
        CK(launch_pack_kmajor(d->torso_deform_w[1], 64, 0, 0, 64, 64, 64, wd1, st));
        CK(launch_pack_rows(d->torso_deform_w[2], 64, 0, 2, 64, 64, wd2, st));
        CK(launch_pack_kmajor(d->torso_canon_w[0], 32 + din, 0, 0, 32, 74, 76, wc0, st));
        CK(launch_pack_kmajor(d->torso_canon_w[1], 32, 0, 0, 32, 32, 32, wc1, st));
        CK(launch_pack_rows(d->torso_canon_w[2], 32, 0, 4, 32, 32, wc2, st));
        CK(launch_pack_tf32(d->torso_deform_w[0], din, d->torso_deform_w[1], d->torso_canon_w[0], 32 + din, d->torso_canon_w[1],
                            (unsigned char *)(base + L.tor_tf32), st));
        m.tor_tf32 = (const unsigned char *)(base + L.tor_tf32);
        m.wd0 = wd0; m.wd1 = wd1; m.wd2 = wd2; m.wc0 = wc0; m.wc1 = wc1; m.wc2 = wc2;
        m.torso_def0_src = d->torso_deform_w[0];
        m.torso_can0_src = d->torso_canon_w[0];
        m.torso_code = d->torso_code;
        m.torso_code_dim = d->torso_code_dim;
        m.density_grid_torso = d->density_grid_torso;
        m.density_thresh_torso = d->density_thresh_torso;
        m.torso_shrink = d->torso_shrink;
    }
    memset(model, 0, sizeof(*model));
    memcpy(model, &m, sizeof(m));
    return GFPP_OK;
}

int gfpp_debug_generate_rays(const float *poses_c2w, uint32_t n_frames, float fx, float fy, float cx, float cy, uint32_t img_h,
                             uint32_t img_w, float *rays_o, float *rays_d, void *stream) {
    if (!poses_c2w || !rays_o || !rays_d || n_frames == 0 || img_h == 0 || img_w == 0)
        return fail(GFPP_ERR_INVALID, "debug_generate_rays: null pointer or empty image%s");
    HeadArgs a;
    memset(&a, 0, sizeof(a));
    a.n_frames = (int)n_frames; a.n_rays = (int)(img_h * img_w);
    a.poses = poses_c2w; a.fx = fx; a.fy = fy; a.cx = cx; a.cy = cy; a.img_w = (int)img_w;
    g_launches = 0;
    CK(launch_dump_rays(a, rays_o, rays_d, (cudaStream_t)stream));
    return GFPP_OK;
}

size_t gfpp_render_workspace_bytes(uint32_t n_frames, uint32_t n_rays, uint32_t max_steps) {
    return work_layout(n_frames, n_rays, max_steps).total;
}

int gfpp_render_frames(const gfpp_model *model, const gfpp_frames *fr, const gfpp_outputs *out, void *workspace,
                       size_t workspace_bytes, void *stream) {
    if (!model || !fr || !out || !workspace) return fail(GFPP_ERR_INVALID, "render_frames: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "render_frames: model handle not initialised by gfpp_model_pack%s");
    if ((!out->rgb_map && !out->rgb_u8 && !out->rgba_u8) || !fr->cond_feat) return fail(GFPP_ERR_INVALID, "render_frames: rgb_map (or rgb_u8) and cond_feat are required%s");
    if ((uintptr_t)out->rgba_u8 & 3) return fail(GFPP_ERR_INVALID, "render_frames: rgba_u8 must be 4-byte aligned%s");
    if (fr->n_frames == 0 || fr->n_rays == 0) return fail(GFPP_ERR_INVALID, "render_frames: empty clip%s");
    if ((uint64_t)fr->n_frames * fr->n_rays >= (1ull << 31)) return fail(GFPP_ERR_UNSUPPORTED, "render_frames: F*N must be < 2^31%s");
    if (fr->max_steps < 1 || fr->max_steps > 4096) return fail(GFPP_ERR_UNSUPPORTED, "render_frames: max_steps must be in 1..4096%s");
    if ((fr->rays_o == nullptr) != (fr->rays_d == nullptr)) return fail(GFPP_ERR_INVALID, "render_frames: rays_o and rays_d go together%s");
    if (!fr->rays_o && (!fr->poses_c2w || fr->img_w == 0 || fr->img_h * fr->img_w != fr->n_rays))
        return fail(GFPP_ERR_INVALID, "render_frames: need rays or (poses_c2w, img_h*img_w == n_rays)%s");
    if (m.has_torso && (!fr->torso_pose6 || !fr->bg_coords)) return fail(GFPP_ERR_INVALID, "render_frames: torso model needs torso_pose6 and bg_coords%s");
    const WorkLayout W = work_layout(fr->n_frames, fr->n_rays, fr->max_steps);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "render_frames: workspace too small%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    g_launches = 0;
    if (g_profile) CKN(cudaEventRecord(g_ev[4], st));
    CKN(cudaMemsetAsync(ws + W.zero_begin, 0, W.zero_end - W.zero_begin, st));

    HeadArgs a;
    memset(&a, 0, sizeof(a));
    a.pos_gm = m.pos_gm; a.amb_gm = m.amb_gm;
    a.pos_tab = m.pos_tab; a.amb_tab = m.amb_tab;
    a.pos_quads = m.pos_quads; a.amb_quads = m.amb_quads;
    a.pos_octs = m.pos_octs; a.amb_octs = m.amb_octs;
    a.wide = m.wide; a.narrow = m.narrow;
    for (int c = 0; c < HEAD_NCHUNK; ++c) { a.chunk_off[c] = m.chunk_off[c]; a.chunk_k[c] = kChunkK[c]; }
    march_const_init(a.mc, m.bound, fr->dt_gamma, fr->max_steps, m.cascade, m.grid_size, m.bitfield);
    a.occ_bounds = m.occ_bounds;
    a.coarse_bits = m.coarse_bits;
    a.coarse_words = m.coarse_words;
    memcpy(a.aabb, m.aabb, sizeof(a.aabb));
    a.min_near = m.min_near; a.density_scale = m.density_scale;
    a.use_occ_box = m.use_occ_box;
    a.n_frames = (int)fr->n_frames; a.n_rays = (int)fr->n_rays;
    a.rays_o = fr->rays_o; a.rays_d = fr->rays_d; a.poses = fr->poses_c2w;
    a.fx = fr->fx; a.fy = fr->fy; a.cx = fr->cx; a.cy = fr->cy; a.img_w = (int)fr->img_w;
    a.cond_feat = fr->cond_feat;
    a.max_steps = (int)fr->max_steps; a.T_thresh = fr->T_thresh;
    a.noises = fr->noises;
    a.image = (float *)(ws + W.image);
    a.wsum = out->weights_sum ? out->weights_sum : (float *)(ws + W.wsum);
    a.depth = out->depth_map ? out->depth_map : (float *)(ws + W.depth);
    a.rays_t = (float *)(ws + W.rays_t);
    a.hist = (int *)(ws + W.hist);
    a.survivors = (int *)(ws + W.survivors);
    int *counters = (int *)(ws + W.counters);
    a.n_survivors = counters + 2;
    a.hits = (uint4 *)(ws + W.hits);
    a.n_hits = counters + 3;
    a.B_total = (int *)(ws + W.B_total);
    a.valid_samples = (int *)(ws + W.valid);

    TorsoArgs t;
    memset(&t, 0, sizeof(t));
    t.has_torso = m.has_torso;
    t.n_frames = a.n_frames; t.n_rays = a.n_rays;
    t.image = a.image; t.wsum = a.wsum;
    t.rgb_map = out->rgb_map;
    t.rgb_u8 = out->rgb_u8;
    t.alpha_map = out->alpha_map;
    t.rgba_u8 = out->rgba_u8;
    t.bg_color = fr->bg_color;
    t.P_count = (int *)(ws + W.pcount);
    if (m.has_torso) {
        t.tor_gm = m.tor_gm; t.tor_tab = m.tor_tab;
        t.w_def0 = m.wd0; t.w_def1 = m.wd1; t.w_def2 = m.wd2; t.w_can0 = m.wc0; t.w_can1 = m.wc1; t.w_can2 = m.wc2;
        t.w_tf32 = m.tor_tf32;
        t.bias_def = (float *)(ws + W.bias_def); t.bias_can = (float *)(ws + W.bias_can);
        t.pose6 = fr->torso_pose6;
        t.density_grid_torso = m.density_grid_torso; t.grid_size = (int)m.grid_size;
        t.density_thresh_torso = m.density_thresh_torso; t.torso_shrink = m.torso_shrink;
        t.bg_coords = fr->bg_coords;
        t.torso_alpha = out->torso_alpha_map; t.torso_rgb = out->torso_rgb_map; t.deform = out->torso_deform;
        CK(launch_torso_frame_bias(t, m.torso_def0_src, m.torso_can0_src, m.torso_code, (int)m.torso_code_dim,
                                   (float *)(ws + W.bias_def), (float *)(ws + W.bias_can), st));
    }

    a.phase_cycles = g_phase;
    a.pass = 1;
    a.cursor = counters + 0;
    CK(launch_ray_setup(a, st));
    // fp16 / robust: the row-owner kernel (head_v2_kernel.cu); GFPP_HEAD_V1 keeps the first-generation fp16 kernel for A/B runs
    const bool use_v2 = m.v2_ok && (m.mlp_precision == 4 || (m.mlp_precision == 1 && getenv("GFPP_HEAD_V1") == nullptr));
    if (m.mlp_precision == 4 && !use_v2) return fail(GFPP_ERR_UNSUPPORTED, "render_frames: robust mode unavailable for this model%s");
    HeadV2Args v2;
    v2.w_stream = m.v2_stream; v2.w_res = m.v2_res; v2.pos_step = m.v2_pos_step;
    v2.cond_hi = (const unsigned char *)(ws + W.bias_amb);
    v2.cond_lo = v2.cond_hi + (size_t)fr->n_frames * 128;
    if (use_v2) CK(launch_cond_images(fr->cond_feat, a.n_frames, ws + W.bias_amb, ws + W.bias_amb + (size_t)fr->n_frames * 128, st));
    if (g_profile) CKN(cudaEventRecord(g_ev[0], st));
    if (m.mlp_precision == 0) CK(launch_head(a, -1, st));
    else if (use_v2) CK(launch_head_v2(a, v2, m.mlp_precision, st));
    else CK(launch_head_tc(a, m.tc, m.mlp_precision, -1, st));
    if (g_profile) CKN(cudaEventRecord(g_ev[1], st));
    CK(launch_schedule(a.hist, a.n_frames, a.n_rays, a.max_steps, a.B_total, st));
    a.pass = 2;
    a.cursor = counters + 1;
    if (m.mlp_precision == 0) CK(launch_head(a, -1, st));
    else if (use_v2) CK(launch_head_v2(a, v2, m.mlp_precision, st));
    else CK(launch_head_tc(a, m.tc, m.mlp_precision, -1, st));
    if (g_profile) CKN(cudaEventRecord(g_ev[2], st));
    CK(launch_epilogue(t, st));
    if (g_profile) CKN(cudaEventRecord(g_ev[3], st));
    if (out->stats) {
        k_write_stats<<<(a.n_frames + 63) / 64, 64, 0, st>>>(a.B_total, a.n_survivors, a.valid_samples, t.P_count,
                                                             a.n_frames, out->stats);
        CK(cudaGetLastError());
    }
    return GFPP_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ (C) super-resolution head (sr_kernel.cu)
namespace {
struct SrHost {
    uint32_t magic;
    const float *conv_in_w, *bias[4], *rgb_w[2], *rgb_b[2];
    const unsigned char *tiles[3];
};
static_assert(sizeof(SrHost) <= sizeof(gfpp_sr_model), "gfpp_sr_model opaque storage too small");
constexpr uint32_t kSrMagic = 0x67667372u;  // "gfsr"
struct SrPacked { size_t conv_in_w, bias[4], rgb_w[2], rgb_b[2], tiles[3], total; };
SrPacked sr_packed_layout() {
    SrPacked L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 1023) / 1024 * 1024; return r; };
    L.conv_in_w = take(27 * 128 * 4);
    const int nb[4] = {128, 128, 64, 64};
    for (int i = 0; i < 4; ++i) L.bias[i] = take((size_t)nb[i] * 4);
    L.rgb_w[0] = take(3 * 128 * 4); L.rgb_w[1] = take(3 * 64 * 4);
    L.rgb_b[0] = take(16); L.rgb_b[1] = take(16);
    for (int l = 0; l < 3; ++l) L.tiles[l] = take((size_t)sr_layer_weight_bytes(l));
    L.total = o;
    return L;
}
struct SrWork { size_t x0a, x0b, img0, x1a, total; };
SrWork sr_work_layout(uint32_t F, uint32_t R) {
    SrWork W;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    const size_t px = (size_t)F * R * R;
    W.x0a = take(px * 128 * 2);
    W.x0b = take(px * 128 * 2);
    W.img0 = take(px * 3 * 4);
    W.x1a = take(px * 4 * 64 * 2);
    W.total = o;
    return W;
}
}  // namespace

extern "C" {

size_t gfpp_sr_packed_bytes(void) { return sr_packed_layout().total; }

int gfpp_sr_pack(const gfpp_sr_desc *d, void *packed, size_t packed_bytes, gfpp_sr_model *model, void *stream) {
    if (!d || !packed || !model) return fail(GFPP_ERR_INVALID, "sr_pack: null pointer%s");
    if (!d->conv_in_w || !d->conv0_w || !d->up_w || !d->conv1_w) return fail(GFPP_ERR_INVALID, "sr_pack: null weight%s");
    for (int i = 0; i < 4; ++i) if (!d->bias[i]) return fail(GFPP_ERR_INVALID, "sr_pack: null bias%s");
    for (int i = 0; i < 2; ++i) if (!d->rgb_w[i] || !d->rgb_b[i]) return fail(GFPP_ERR_INVALID, "sr_pack: null toRGB weight%s");
    const SrPacked L = sr_packed_layout();
    if (packed_bytes < L.total) return fail(GFPP_ERR_WORKSPACE, "sr_pack: packed buffer too small%s");
    if (((uintptr_t)packed & 1023u) != 0) return fail(GFPP_ERR_INVALID, "sr_pack: packed buffer must be 1024-byte aligned%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *base = (char *)packed;
    g_launches = 0;
    CKN(cudaMemsetAsync(packed, 0, L.total, st));
    CKN(cudaMemcpyAsync(base + L.conv_in_w, d->conv_in_w, 27 * 128 * 4, cudaMemcpyDeviceToDevice, st));
    const int nb[4] = {128, 128, 64, 64};
    for (int i = 0; i < 4; ++i) CKN(cudaMemcpyAsync(base + L.bias[i], d->bias[i], (size_t)nb[i] * 4, cudaMemcpyDeviceToDevice, st));
    CKN(cudaMemcpyAsync(base + L.rgb_w[0], d->rgb_w[0], 3 * 128 * 4, cudaMemcpyDeviceToDevice, st));
    CKN(cudaMemcpyAsync(base + L.rgb_w[1], d->rgb_w[1], 3 * 64 * 4, cudaMemcpyDeviceToDevice, st));
    CKN(cudaMemcpyAsync(base + L.rgb_b[0], d->rgb_b[0], 12, cudaMemcpyDeviceToDevice, st));
    CKN(cudaMemcpyAsync(base + L.rgb_b[1], d->rgb_b[1], 12, cudaMemcpyDeviceToDevice, st));
    // GEMM matrices [N_total][9 * C_in] -> fp16 GMMA K-major SW128 tiles in the kernels' streaming order:
    // chunk c covers k in [64c, 64c + 64) (tap c / CB, channel block c % CB); inside a chunk one tile per N-block
    const float *mat[3] = {d->conv0_w, d->up_w, d->conv1_w};
    for (int l = 0; l < 3; ++l) {
        const int ld = 9 * sr_layer_cin(l), nrows = sr_layer_nrows(l);
        unsigned char *dst = (unsigned char *)(base + L.tiles[l]);
        for (int c = 0; c < sr_layer_nchunk(l); ++c)
            for (int b = 0; b < sr_layer_nb(l); ++b)
                CK(launch_pack_tc_tile(mat[l], ld, b * nrows, c * 64, nrows, 64, 0, 0, 0,
                                       dst + ((size_t)c * sr_layer_nb(l) + b) * nrows * 128, nullptr, st));
    }
    SrHost m;
    memset(&m, 0, sizeof(m));
    m.magic = kSrMagic;
    m.conv_in_w = (const float *)(base + L.conv_in_w);
    for (int i = 0; i < 4; ++i) m.bias[i] = (const float *)(base + L.bias[i]);
    for (int i = 0; i < 2; ++i) { m.rgb_w[i] = (const float *)(base + L.rgb_w[i]); m.rgb_b[i] = (const float *)(base + L.rgb_b[i]); }
    for (int l = 0; l < 3; ++l) m.tiles[l] = (const unsigned char *)(base + L.tiles[l]);
    memset(model, 0, sizeof(*model));
    memcpy(model, &m, sizeof(m));
    return GFPP_OK;
}

size_t gfpp_sr_workspace_bytes(uint32_t n_frames, uint32_t in_res) { return sr_work_layout(n_frames, in_res).total; }

}  // extern "C"

// gfpp_sr_forward (out, clamp01) and gfpp_sr_forward_video (out and/or out_u8, always clamped): `who` names the entry point in errors
static int sr_forward_impl(const char *who, const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in,
                           const float *const noise[4], uint32_t noise_per_frame, float *out, uint8_t *out_u8, int clamp01, void *workspace,
                           size_t workspace_bytes, void *stream) {
    if (!model || !rgb_in || (!out && !out_u8) || !workspace) return fail(GFPP_ERR_INVALID, "%s: null pointer", who);
    if (((uintptr_t)out_u8 & 3u) != 0) return fail(GFPP_ERR_INVALID, "%s: out_u8 must be 4-byte aligned", who);
    SrHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kSrMagic) return fail(GFPP_ERR_INVALID, "%s: model handle not initialised by gfpp_sr_pack", who);
    if (n_frames == 0 || in_res == 0 || in_res % 128 != 0 || in_res > 1024) return fail(GFPP_ERR_UNSUPPORTED, "%s: in_res must be a multiple of 128 (256 in the reference)", who);
    if ((uint64_t)n_frames * in_res * in_res * 4 >= (1ull << 31)) return fail(GFPP_ERR_UNSUPPORTED, "%s: too many frames per call", who);
    const SrWork W = sr_work_layout(n_frames, in_res);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "%s: workspace too small", who);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    const int F = (int)n_frames, R = (int)in_res;
    const long long lo = noise_per_frame ? (long long)R * R : 0, hi = noise_per_frame ? 4ll * R * R : 0;
    g_launches = 0;
    SrConvInArgs ci;
    memset(&ci, 0, sizeof(ci));
    ci.in = rgb_in; ci.F = F; ci.H = R; ci.W = R; ci.w = m.conv_in_w; ci.bias = m.bias[0];
    ci.noise = noise ? noise[0] : nullptr; ci.noise_fstride = lo; ci.out = (__half *)(ws + W.x0a);
    CK(launch_sr_conv_in(ci, st));
    SrConvArgs a;
    memset(&a, 0, sizeof(a));
    a.in = (const __half *)(ws + W.x0a); a.F = F; a.H = R; a.W = R; a.wt = m.tiles[0]; a.bias = m.bias[1];
    a.noise = noise ? noise[1] : nullptr; a.noise_fstride = lo; a.out = (__half *)(ws + W.x0b);
    a.rgb_w = m.rgb_w[0]; a.rgb_b = m.rgb_b[0]; a.img_in = rgb_in; a.img_out = (float *)(ws + W.img0);
    CK(launch_sr_conv(0, a, st));
    memset(&a, 0, sizeof(a));
    a.in = (const __half *)(ws + W.x0b); a.F = F; a.H = R; a.W = R; a.wt = m.tiles[1]; a.bias = m.bias[2];
    a.noise = noise ? noise[2] : nullptr; a.noise_fstride = hi; a.out = (__half *)(ws + W.x1a);
    CK(launch_sr_conv(1, a, st));
    memset(&a, 0, sizeof(a));
    a.in = (const __half *)(ws + W.x1a); a.F = F; a.H = 2 * R; a.W = 2 * R; a.wt = m.tiles[2]; a.bias = m.bias[3];
    a.noise = noise ? noise[3] : nullptr; a.noise_fstride = hi;
    a.rgb_w = m.rgb_w[1]; a.rgb_b = m.rgb_b[1]; a.img_in = (const float *)(ws + W.img0); a.img_out = out; a.clamp01 = clamp01;
    a.img_u8 = out_u8;
    CK(launch_sr_conv(2, a, st));
    return GFPP_OK;
}

extern "C" {

int gfpp_sr_forward(const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in, const float *const noise[4],
                    uint32_t noise_per_frame, float *out, int clamp01, void *workspace, size_t workspace_bytes, void *stream) {
    if (!out) return fail(GFPP_ERR_INVALID, "sr_forward: null pointer%s");
    return sr_forward_impl("sr_forward", model, n_frames, in_res, rgb_in, noise, noise_per_frame, out, nullptr, clamp01, workspace,
                           workspace_bytes, stream);
}

int gfpp_sr_forward_video(const gfpp_sr_model *model, uint32_t n_frames, uint32_t in_res, const float *rgb_in, const float *const noise[4],
                          uint32_t noise_per_frame, float *out, uint8_t *out_u8, void *workspace, size_t workspace_bytes, void *stream) {
    return sr_forward_impl("sr_forward_video", model, n_frames, in_res, rgb_in, noise, noise_per_frame, out, out_u8, 1, workspace,
                           workspace_bytes, stream);
}

}  // extern "C"

// ------------------------------------------------------------------ (C) torso field of the torso-SR checkpoints (torso_sr_kernel.cu)
namespace {
struct TorsoSrHost {
    uint32_t magic;
    int head_aware;
    GridMeta tor_gm;
    const float2 *tor_tab;
    const float *wd0, *wd1, *wd2, *wc0, *wc1, *wc2, *ha;
    const float *def0_src, *can0_src, *code;     // originals (the per-frame bias fold reads them)
    uint32_t code_dim;
    const float *density_grid_torso;
    uint32_t grid_size;
    float density_thresh_torso, torso_shrink;
};
static_assert(sizeof(TorsoSrHost) <= sizeof(gfpp_torso_sr_model), "gfpp_torso_sr_model opaque storage too small");
constexpr uint32_t kTorsoSrMagic = 0x67667473u;  // "gfts"
struct TorsoSrPacked { size_t wd0, wd1, wd2, wc0, wc1, wc2, ha, total; };
TorsoSrPacked torso_sr_packed_layout() {
    TorsoSrPacked L;
    size_t o = 0;
    auto take = [&](size_t floats) { size_t r = o; o += (floats * 4 + 255) / 256 * 256; return r; };
    L.wd0 = take(TORSO_SR_KD0 * 64); L.wd1 = take(64 * 64); L.wd2 = take(2 * 64);
    L.wc0 = take(TORSO_SR_KC0 * 32); L.wc1 = take(32 * 32); L.wc2 = take(4 * 32);
    L.ha = take(TORSO_SR_HA_FLOATS);
    L.total = o;
    return L;
}
struct TorsoSrWork { size_t bias_def, bias_can, pcount, total; };
TorsoSrWork torso_sr_work_layout(uint32_t F) {
    TorsoSrWork W;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    W.bias_def = take((size_t)F * 64 * 4);
    W.bias_can = take((size_t)F * 32 * 4);
    W.pcount = take((size_t)F * 4);
    W.total = o;
    return W;
}
__global__ void k_copy_ints(const int *src, int n, int32_t *dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}
}  // namespace

extern "C" {

size_t gfpp_torso_sr_packed_bytes(void) { return torso_sr_packed_layout().total; }

int gfpp_torso_sr_pack(const gfpp_torso_sr_desc *d, void *packed, size_t packed_bytes, gfpp_torso_sr_model *model, void *stream) {
    if (!d || !packed || !model) return fail(GFPP_ERR_INVALID, "torso_sr_pack: null pointer%s");
    const TorsoSrPacked L = torso_sr_packed_layout();
    if (packed_bytes < L.total) return fail(GFPP_ERR_WORKSPACE, "torso_sr_pack: packed buffer too small%s");
    for (int i = 0; i < 3; ++i)
        if (!d->torso_deform_w[i] || !d->torso_canon_w[i]) return fail(GFPP_ERR_INVALID, "torso_sr_pack: null torso weight%s");
    if (!d->density_grid_torso || !d->torso_grid.embeddings || !d->torso_grid.offsets_host) return fail(GFPP_ERR_INVALID, "torso_sr_pack: null grid%s");
    if (d->torso_code_dim > 10 || (d->torso_code_dim > 0 && !d->torso_code)) return fail(GFPP_ERR_UNSUPPORTED, "torso_sr_pack: torso_code_dim <= 10 (with a code pointer)%s");
    if (d->head_aware)
        for (int i = 0; i < 3; ++i)
            if (!d->ha_w[i] || !d->ha_b[i]) return fail(GFPP_ERR_INVALID, "torso_sr_pack: null head-aware encoder weight%s");
    TorsoSrHost m;
    memset(&m, 0, sizeof(m));
    m.magic = kTorsoSrMagic;
    if (d->torso_grid.num_levels != 16 ||
        fill_grid_meta(m.tor_gm, d->torso_grid.offsets_host, d->torso_grid.input_dim, d->torso_grid.num_levels, d->torso_grid.log2_per_level_scale,
                       d->torso_grid.base_resolution, d->torso_grid.gridtype, d->torso_grid.align_corners, d->torso_grid.interp) != 0 ||
        m.tor_gm.dim != 2)
        return fail(GFPP_ERR_UNSUPPORTED, "torso_sr_pack: the torso grid must be 2-D with 16 levels x 2 features%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *base = (char *)packed;
    g_launches = 0;
    CKN(cudaMemsetAsync(packed, 0, L.total, st));
    const int ha = d->head_aware ? 1 : 0;
    const int nh = (int)d->torso_code_dim + 126;
    const int din = 42 + nh + (ha ? 16 : 0);
    float *wd0 = (float *)(base + L.wd0), *wd1 = (float *)(base + L.wd1), *wd2 = (float *)(base + L.wd2);
    float *wc0 = (float *)(base + L.wc0), *wc1 = (float *)(base + L.wc1), *wc2 = (float *)(base + L.wc2), *hab = (float *)(base + L.ha);
    // input columns of the reference layers: deform [enc_x 42 | code | lm 126 | head-aware 16], canonical [grid 32 | the same]
    CK(launch_pack_kmajor(d->torso_deform_w[0], din, 0, 0, 64, 42, 42, wd0, st));
    CK(launch_pack_kmajor(d->torso_deform_w[0], din, 0, 42 + nh, 64, ha ? 16 : 0, 18, wd0 + 42 * 64, st));
    CK(launch_pack_kmajor(d->torso_deform_w[1], 64, 0, 0, 64, 64, 64, wd1, st));
    CK(launch_pack_rows(d->torso_deform_w[2], 64, 0, 2, 64, 64, wd2, st));
    CK(launch_pack_kmajor(d->torso_canon_w[0], 32 + din, 0, 0, 32, 74, 74, wc0, st));
    CK(launch_pack_kmajor(d->torso_canon_w[0], 32 + din, 0, 74 + nh, 32, ha ? 16 : 0, 18, wc0 + 74 * 32, st));
    CK(launch_pack_kmajor(d->torso_canon_w[1], 32, 0, 0, 32, 32, 32, wc1, st));
    CK(launch_pack_rows(d->torso_canon_w[2], 32, 0, 4, 32, 32, wc2, st));
    if (ha) {
        CK(launch_pack_kmajor(d->ha_w[0], 4, 0, 0, 16, 4, 4, hab + TORSO_SR_HA_W0, st));
        CK(launch_pack_kmajor(d->ha_w[1], 16, 0, 0, 32, 16, 16, hab + TORSO_SR_HA_W1, st));
        CK(launch_pack_kmajor(d->ha_w[2], 32, 0, 0, 16, 32, 32, hab + TORSO_SR_HA_W2, st));
        CKN(cudaMemcpyAsync(hab + TORSO_SR_HA_B0, d->ha_b[0], 16 * 4, cudaMemcpyDeviceToDevice, st));
        CKN(cudaMemcpyAsync(hab + TORSO_SR_HA_B1, d->ha_b[1], 32 * 4, cudaMemcpyDeviceToDevice, st));
        CKN(cudaMemcpyAsync(hab + TORSO_SR_HA_B2, d->ha_b[2], 16 * 4, cudaMemcpyDeviceToDevice, st));
    }
    m.head_aware = ha;
    m.tor_tab = (const float2 *)d->torso_grid.embeddings;
    m.wd0 = wd0; m.wd1 = wd1; m.wd2 = wd2; m.wc0 = wc0; m.wc1 = wc1; m.wc2 = wc2; m.ha = ha ? hab : nullptr;
    m.def0_src = d->torso_deform_w[0]; m.can0_src = d->torso_canon_w[0]; m.code = d->torso_code; m.code_dim = d->torso_code_dim;
    m.density_grid_torso = d->density_grid_torso; m.grid_size = d->grid_size;
    m.density_thresh_torso = d->density_thresh_torso; m.torso_shrink = d->torso_shrink;
    memset(model, 0, sizeof(*model));
    memcpy(model, &m, sizeof(m));
    return GFPP_OK;
}

size_t gfpp_torso_sr_workspace_bytes(uint32_t n_frames) { return torso_sr_work_layout(n_frames).total; }

int gfpp_torso_sr_composite(const gfpp_torso_sr_model *model, const gfpp_torso_sr_frames *fr, float *rgb_map, float *torso_alpha_map,
                            float *torso_rgb_map, float *torso_deform, int32_t *torso_pixels, void *workspace, size_t workspace_bytes,
                            void *stream) {
    if (!model || !fr || !rgb_map || !workspace) return fail(GFPP_ERR_INVALID, "torso_sr_composite: null pointer%s");
    TorsoSrHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kTorsoSrMagic) return fail(GFPP_ERR_INVALID, "torso_sr_composite: model handle not initialised by gfpp_torso_sr_pack%s");
    if (!fr->image || !fr->weights_sum || !fr->lm68 || !fr->bg_coords) return fail(GFPP_ERR_INVALID, "torso_sr_composite: image, weights_sum, lm68 and bg_coords are required%s");
    if (fr->n_frames == 0 || fr->n_rays == 0) return fail(GFPP_ERR_INVALID, "torso_sr_composite: empty clip%s");
    if ((uint64_t)fr->n_frames * fr->n_rays >= (1ull << 31)) return fail(GFPP_ERR_UNSUPPORTED, "torso_sr_composite: F*N must be < 2^31%s");
    const TorsoSrWork W = torso_sr_work_layout(fr->n_frames);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "torso_sr_composite: workspace too small%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    g_launches = 0;
    CKN(cudaMemsetAsync(ws + W.pcount, 0, (size_t)fr->n_frames * 4, st));
    CK(launch_torso_sr_frame_bias(fr->lm68, (int)fr->n_frames, m.def0_src, m.can0_src, m.code, (int)m.code_dim, m.head_aware,
                                  (float *)(ws + W.bias_def), (float *)(ws + W.bias_can), st));
    TorsoSrArgs t;
    memset(&t, 0, sizeof(t));
    t.tor_gm = m.tor_gm; t.tor_tab = m.tor_tab;
    t.w_def0 = m.wd0; t.w_def1 = m.wd1; t.w_def2 = m.wd2; t.w_can0 = m.wc0; t.w_can1 = m.wc1; t.w_can2 = m.wc2; t.ha = m.ha;
    t.bias_def = (const float *)(ws + W.bias_def); t.bias_can = (const float *)(ws + W.bias_can);
    t.density_grid_torso = m.density_grid_torso; t.grid_size = (int)m.grid_size;
    t.density_thresh_torso = m.density_thresh_torso; t.torso_shrink = m.torso_shrink;
    t.bg_coords = fr->bg_coords; t.bg_color = fr->bg_color;
    t.n_frames = (int)fr->n_frames; t.n_rays = (int)fr->n_rays;
    t.image = fr->image; t.wsum = fr->weights_sum;
    t.rgb_map = rgb_map; t.torso_alpha = torso_alpha_map; t.torso_rgb = torso_rgb_map; t.deform = torso_deform;
    t.P_count = (int *)(ws + W.pcount);
    CK(launch_torso_sr(t, st));
    if (torso_pixels) {
        k_copy_ints<<<(fr->n_frames + 127) / 128, 128, 0, st>>>(t.P_count, (int)fr->n_frames, torso_pixels);
        CK(cudaGetLastError());
    }
    return GFPP_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ (D) training-side ops (train_kernels.cu)
extern "C" {

size_t gfpp_march_rays_train_scratch_bytes(uint32_t N) { return march_train_scratch_bytes(N); }

int gfpp_march_rays_train(const float *rays_o, const float *rays_d, const uint8_t *grid, float bound, float dt_gamma, uint32_t max_steps,
                          uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float *nears, const float *fars, float *xyzs, float *dirs,
                          float *deltas, int32_t *rays, int32_t *counter, const float *noises, void *scratch, size_t scratch_bytes,
                          void *stream) {
    if (!rays_o || !rays_d || !grid || !nears || !fars || !xyzs || !dirs || !deltas || !rays || !counter || !noises || !scratch)
        return fail(GFPP_ERR_INVALID, "march_rays_train: null pointer%s");
    if (C < 1 || C > 8 || H < 1 || H > 1024 || max_steps < 1) return fail(GFPP_ERR_INVALID, "march_rays_train: bad C/H/max_steps%s");
    if (scratch_bytes < march_train_scratch_bytes(N)) return fail(GFPP_ERR_WORKSPACE, "march_rays_train: scratch too small%s");
    if (N > (1u << 24)) return fail(GFPP_ERR_UNSUPPORTED, "march_rays_train: N <= 2^24 rays per call%s");
    MarchConst mc;
    march_const_init(mc, bound, dt_gamma, max_steps, C, H, grid);
    g_launches = 0;
    int nl = 0;
    CKN(launch_march_rays_train(mc, rays_o, rays_d, nears, fars, noises, N, M, max_steps, xyzs, dirs, deltas, (int *)rays, (int *)counter,
                                (int *)scratch, &nl, (cudaStream_t)stream));
    g_launches = nl;
    return GFPP_OK;
}

int gfpp_march_rays_train_backward(const float *grad_xyzs, const float *grad_dirs, const int32_t *rays, const float *deltas, uint32_t N,
                                   uint32_t M, float *grad_rays_o, float *grad_rays_d, void *stream) {
    if (!grad_xyzs || !grad_dirs || !rays || !deltas || !grad_rays_o || !grad_rays_d) return fail(GFPP_ERR_INVALID, "march_rays_train_backward: null pointer%s");
    g_launches = 0;
    CK(launch_march_rays_train_backward(grad_xyzs, grad_dirs, (const int *)rays, deltas, N, M, grad_rays_o, grad_rays_d, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_composite_rays_train_forward(const float *sigmas, const float *rgbs, const float *ambient, const float *deltas, const int32_t *rays,
                                      uint32_t M, uint32_t N, float T_thresh, float *weights_sum, float *ambient_sum, float *depth,
                                      float *image, void *stream) {
    if (!sigmas || !rgbs || !ambient || !deltas || !rays || !weights_sum || !ambient_sum || !depth || !image)
        return fail(GFPP_ERR_INVALID, "composite_rays_train_forward: null pointer%s");
    g_launches = 0;
    CK(launch_composite_train_forward(sigmas, rgbs, ambient, deltas, (const int *)rays, M, N, T_thresh, weights_sum, ambient_sum, depth, image,
                                      (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_composite_rays_train_backward(const float *grad_weights_sum, const float *grad_ambient_sum, const float *grad_image,
                                       const float *sigmas, const float *rgbs, const float *ambient, const float *deltas, const int32_t *rays,
                                       const float *weights_sum, const float *ambient_sum, const float *image, uint32_t M, uint32_t N,
                                       float T_thresh, float *grad_sigmas, float *grad_rgbs, float *grad_ambient, void *stream) {
    if (!grad_weights_sum || !grad_ambient_sum || !grad_image || !sigmas || !rgbs || !ambient || !deltas || !rays || !weights_sum || !ambient_sum ||
        !image || !grad_sigmas || !grad_rgbs || !grad_ambient)
        return fail(GFPP_ERR_INVALID, "composite_rays_train_backward: null pointer%s");
    g_launches = 0;
    CK(launch_composite_train_backward(grad_weights_sum, grad_ambient_sum, grad_image, sigmas, rgbs, ambient, deltas, (const int *)rays,
                                       weights_sum, ambient_sum, image, M, N, T_thresh, grad_sigmas, grad_rgbs, grad_ambient, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_grid_encode_forward_dydx(const float *inputs, const float *embeddings, const int32_t *offsets_host, float *outputs, uint32_t B,
                                  uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, float *dy_dx, uint32_t gridtype, int align_corners,
                                  uint32_t interp, void *stream) {
    if (!inputs || !embeddings || !offsets_host || !outputs || !dy_dx) return fail(GFPP_ERR_INVALID, "grid_encode_forward_dydx: null pointer%s");
    if (C != 2) return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: this build supports C == 2 only%s");
    GridMeta gm;
    if (fill_grid_meta(gm, offsets_host, D, L, S, H, gridtype, align_corners, interp) != 0)
        return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: D must be 2 or 3 and L <= 16%s");
    g_launches = 0;
    CK(launch_grid_encode_dydx(gm, inputs, embeddings, outputs, dy_dx, B, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_grid_encode_backward(const float *grad, const float *inputs, const float *embeddings, const int32_t *offsets_host,
                              float *grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, const float *dy_dx,
                              float *grad_inputs, uint32_t gridtype, int align_corners, uint32_t interp, void *stream) {
    (void)embeddings;   // the reference passes the table too (gridencoder.h:13) but only uses its dtype
    if (!grad || !inputs || !offsets_host || !grad_embeddings) return fail(GFPP_ERR_INVALID, "grid_encode_backward: null pointer%s");
    if ((dy_dx == nullptr) != (grad_inputs == nullptr)) return fail(GFPP_ERR_INVALID, "grid_encode_backward: dy_dx and grad_inputs go together%s");
    if (C != 2) return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: this build supports C == 2 only%s");
    GridMeta gm;
    if (fill_grid_meta(gm, offsets_host, D, L, S, H, gridtype, align_corners, interp) != 0)
        return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: D must be 2 or 3 and L <= 16%s");
    g_launches = 0;
    int nl = 0;
    CKN(launch_grid_backward(gm, grad, inputs, grad_embeddings, dy_dx, grad_inputs, B, &nl, (cudaStream_t)stream));
    g_launches = nl;
    return GFPP_OK;
}

int gfpp_grad_total_variation(const float *inputs, const float *embeddings, float *grad, const int32_t *offsets_host, float weight, uint32_t B,
                              uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, uint32_t gridtype, int align_corners, void *stream) {
    if (!inputs || !embeddings || !grad || !offsets_host) return fail(GFPP_ERR_INVALID, "grad_total_variation: null pointer%s");
    if (C != 2) return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: this build supports C == 2 only%s");
    GridMeta gm;
    if (fill_grid_meta(gm, offsets_host, D, L, S, H, gridtype, align_corners, 0) != 0)
        return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: D must be 2 or 3 and L <= 16%s");
    g_launches = 0;
    CK(launch_grad_tv(gm, inputs, embeddings, grad, weight, B, (cudaStream_t)stream));
    return GFPP_OK;
}

// ---------------------------------------------------------------- (L) half-table grid encoder
namespace {

// the shape checks of the fp32 ops (fill_grid_meta: D, L, non-empty levels), then the raw level layout for the device
int half_grid_args(HalfGridArgs &g, const int32_t *offsets, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, uint32_t gridtype,
                   int align_corners, uint32_t interp) {
    if (C != 2) return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: this build supports C == 2 only%s");
    GridMeta gm;
    if (fill_grid_meta(gm, offsets, D, L, S, H, gridtype, align_corners, interp) != 0)
        return fail(GFPP_ERR_UNSUPPORTED, "GridEncoding: D must be 2 or 3 and L <= 16%s");
    memset(&g, 0, sizeof(g));
    for (uint32_t l = 0; l <= L; ++l) g.offset[l] = (uint32_t)offsets[l];
    g.L = L;
    g.S = S;
    g.H = H;
    g.gridtype = gridtype;
    g.align_corners = align_corners ? 1u : 0u;
    g.interp = interp;
    return GFPP_OK;
}

bool misaligned4(const void *p) { return ((uintptr_t)p & 3u) != 0; }

}  // namespace

int gfpp_grid_encode_forward_half(const float *inputs, const uint16_t *embeddings, const int32_t *offsets_host, uint16_t *outputs,
                                  uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, uint16_t *dy_dx, uint32_t gridtype,
                                  int align_corners, uint32_t interp, void *stream) {
    if (!inputs || !embeddings || !offsets_host || !outputs) return fail(GFPP_ERR_INVALID, "grid_encode_forward_half: null pointer%s");
    HalfGridArgs g;
    const int rc = half_grid_args(g, offsets_host, D, C, L, S, H, gridtype, align_corners, interp);
    if (rc != GFPP_OK) return rc;
    if (misaligned4(embeddings) || misaligned4(outputs) || misaligned4(dy_dx))
        return fail(GFPP_ERR_INVALID, "grid_encode_forward_half: half2 buffers must be 4-byte aligned%s");
    g_launches = 0;
    if (B == 0) return GFPP_OK;
    CK(launch_grid_half_forward(g, D, inputs, embeddings, outputs, dy_dx, B, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_grid_encode_backward_half(const uint16_t *grad, const float *inputs, const uint16_t *embeddings, const int32_t *offsets_host,
                                   uint16_t *grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
                                   const uint16_t *dy_dx, uint16_t *grad_inputs, uint32_t gridtype, int align_corners, uint32_t interp,
                                   void *stream) {
    (void)embeddings;   // only its dtype matters to the reference (gridencoder.cu:497)
    if (!grad || !inputs || !offsets_host || !grad_embeddings) return fail(GFPP_ERR_INVALID, "grid_encode_backward_half: null pointer%s");
    if ((dy_dx == nullptr) != (grad_inputs == nullptr))
        return fail(GFPP_ERR_INVALID, "grid_encode_backward_half: dy_dx and grad_inputs go together%s");
    HalfGridArgs g;
    const int rc = half_grid_args(g, offsets_host, D, C, L, S, H, gridtype, align_corners, interp);
    if (rc != GFPP_OK) return rc;
    if (misaligned4(grad) || misaligned4(grad_embeddings) || misaligned4(dy_dx))
        return fail(GFPP_ERR_INVALID, "grid_encode_backward_half: half2 buffers must be 4-byte aligned%s");
    g_launches = 0;
    if (B == 0) return GFPP_OK;
    int nl = 0;
    CKN(launch_grid_half_backward(g, D, grad, inputs, grad_embeddings, dy_dx, grad_inputs, B, &nl, (cudaStream_t)stream));
    g_launches = nl;
    return GFPP_OK;
}

int gfpp_packbits(const float *grid, uint32_t N, float density_thresh, uint8_t *bitfield, void *stream) {
    if (!grid || !bitfield) return fail(GFPP_ERR_INVALID, "packbits: null pointer%s");
    if (((uintptr_t)grid & 15u) != 0) return fail(GFPP_ERR_INVALID, "packbits: grid must be 16-byte aligned%s");
    g_launches = 0;
    CK(launch_packbits(grid, N, density_thresh, bitfield, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_morton3D(const int32_t *coords, uint32_t N, int32_t *indices, void *stream) {
    if (!coords || !indices) return fail(GFPP_ERR_INVALID, "morton3D: null pointer%s");
    g_launches = 0;
    CK(launch_morton3D((const int *)coords, N, (int *)indices, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_morton3D_invert(const int32_t *indices, uint32_t N, int32_t *coords, void *stream) {
    if (!coords || !indices) return fail(GFPP_ERR_INVALID, "morton3D_invert: null pointer%s");
    g_launches = 0;
    CK(launch_morton3D_invert((const int *)indices, N, (int *)coords, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_morton3D_dilation(const float *grid, uint32_t C, uint32_t H, float *grid_dilation, void *stream) {
    if (!grid || !grid_dilation) return fail(GFPP_ERR_INVALID, "morton3D_dilation: null pointer%s");
    if (C < 1 || C > 8 || H < 1 || H > 1024) return fail(GFPP_ERR_INVALID, "morton3D_dilation: bad C/H%s");
    g_launches = 0;
    CK(launch_morton3D_dilation(grid, C, H, grid_dilation, (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_sph_from_ray(const float *rays_o, const float *rays_d, float radius, uint32_t N, float *coords, void *stream) {
    if (!rays_o || !rays_d || !coords) return fail(GFPP_ERR_INVALID, "sph_from_ray: null pointer%s");
    g_launches = 0;
    CK(launch_sph_from_ray(rays_o, rays_d, radius, N, coords, (cudaStream_t)stream));
    return GFPP_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ (E) occupancy-grid maintenance (head_kernel.cu: k_density; grid_kernels.cu)
namespace {

bool grid_shape_ok(uint32_t C, uint32_t H) {
    // Morton codes below H^3 decode to cells inside the grid only for a power-of-two H (the reference assumes one too)
    return C >= 1 && C <= 8 && H >= 8 && H <= 512 && (H & (H - 1)) == 0 && (uint64_t)C * H * H * H <= (1ull << 30);
}

struct GridWork {
    size_t tmp, partial, thresh, total;
};

GridWork grid_work_layout(uint32_t C, uint32_t H) {
    GridWork W;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    W.tmp = take((size_t)C * H * H * H * 4);
    W.partial = take((size_t)dilate_ema_blocks(C, H) * 8);
    W.thresh = take(4);
    W.total = o;
    return W;
}

// the head field of a packed model, for k_density: fp32 weight chunks and fp32 tables (quads where the mode packed them)
HeadArgs density_head_args(const ModelHost &m) {
    HeadArgs a;
    memset(&a, 0, sizeof(a));
    a.pos_gm = m.pos_gm; a.amb_gm = m.amb_gm;
    a.pos_tab = m.pos_tab; a.amb_tab = m.amb_tab;
    a.pos_quads = m.pos_quads; a.amb_quads = m.amb_quads;
    a.pos_octs = m.pos_octs; a.amb_octs = m.amb_octs;
    a.wide = m.wide; a.narrow = m.narrow;
    for (int c = 0; c < HEAD_NCHUNK; ++c) { a.chunk_off[c] = m.chunk_off[c]; a.chunk_k[c] = kChunkK[c]; }
    return a;
}

// the field the model's mode renders where a query kernel for it exists: fp16 -> wgmma over the fp16 operand images and oct tables;
// fp32 / bf16x3 / bf16 / robust -> the fp32 FFMA field (robust renders a split-precision approximation of it, DESIGN.md section 6)
cudaError_t launch_density_for(const ModelHost &m, const DensityArgs &d, cudaStream_t st) {
    const HeadArgs a = density_head_args(m);
    if (m.mlp_precision == 1 && m.tc.w_hi && m.pos_octs && m.amb_octs) return launch_density_tc(a, m.tc, d, st);
    return launch_density(a, d, st);
}

// per cascade c: bound_c = min(2^c, bound), hgs_c = bound_c / H in double as the reference's Python does (renderer.py:253-254, 171-172)
void cascade_constants(double bound, uint32_t C, uint32_t H, float *scale, float *hgs, float *pad) {
    for (uint32_t c = 0; c < 8; ++c) {
        const double bc = c < C ? fmin(ldexp(1.0, (int)c), bound) : 0.0, h = bc / (double)H;
        scale[c] = (float)(bc - h);
        if (hgs) hgs[c] = (float)h;
        if (pad) pad[c] = (float)(h * 2.0);
    }
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace

extern "C" {

int gfpp_density_query(const gfpp_model *model, const float *xyzs, uint32_t n, const float *cond_feat, float *sigma, float *geo_feat,
                       void *stream) {
    if (!model || !xyzs || !cond_feat || !sigma) return fail(GFPP_ERR_INVALID, "density_query: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "density_query: model handle not initialised by gfpp_model_pack%s");
    if (!aligned16(cond_feat) || (geo_feat && !aligned16(geo_feat)))
        return fail(GFPP_ERR_INVALID, "density_query: cond_feat and geo_feat must be 16-byte aligned%s");
    if (n >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "density_query: n must be < 2^31%s");
    DensityArgs d;
    memset(&d, 0, sizeof(d));
    d.n = n; d.xyzs = xyzs; d.cond = cond_feat; d.bound = m.bound;
    d.sigma = sigma; d.geo = geo_feat; d.out_scale = 1.0f;
    g_launches = 0;
    CK(launch_density_for(m, d, (cudaStream_t)stream));
    return GFPP_OK;
}

size_t gfpp_density_grid_workspace_bytes(uint32_t cascade, uint32_t grid_size) {
    return grid_shape_ok(cascade, grid_size) ? grid_work_layout(cascade, grid_size).total : 0;
}

int gfpp_density_grid_update(const gfpp_model *model, const float *cond_feat, const float *noise, float decay, float density_thresh,
                             float *density_grid, float *mean_out, float *tmp_grid, void *workspace, size_t workspace_bytes, void *stream) {
    if (!model || !cond_feat || !noise || !density_grid || !mean_out || !workspace)
        return fail(GFPP_ERR_INVALID, "density_grid_update: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "density_grid_update: model handle not initialised by gfpp_model_pack%s");
    const uint32_t C = m.cascade, H = m.grid_size;
    if (!grid_shape_ok(C, H))
        return fail(GFPP_ERR_UNSUPPORTED, "density_grid_update: needs cascade 1..8, grid_size a power of two in 8..512, C*H^3 <= 2^30%s");
    if (!aligned16(cond_feat) || !aligned16(density_grid) || (tmp_grid && !aligned16(tmp_grid)))
        return fail(GFPP_ERR_INVALID, "density_grid_update: cond_feat, density_grid and tmp_grid must be 16-byte aligned%s");
    const GridWork W = grid_work_layout(C, H);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "density_grid_update: workspace too small%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    float *tmp = tmp_grid ? tmp_grid : (float *)(ws + W.tmp);
    const uint32_t H3 = H * H * H;
    DensityArgs d;
    memset(&d, 0, sizeof(d));
    d.n = C * H3; d.cond = cond_feat; d.bound = m.bound;
    d.grid_size = H; d.noise = noise;
    cascade_constants((double)m.bound, C, H, d.cell_scale, d.hgs, nullptr);
    d.sigma = tmp; d.out_scale = m.density_scale;
    g_launches = 0;
    CK(launch_density_for(m, d, st));
    uint8_t *bits = const_cast<uint8_t *>(m.bitfield);
    int nl = 0;
    const cudaError_t et = launch_grid_refresh_tail(tmp, C, H, decay, density_thresh, density_grid, (double *)(ws + W.partial), mean_out,
                                                    (float *)(ws + W.thresh), bits, &nl, st);
    g_launches += nl;
    if (et != cudaSuccess) return fail(GFPP_ERR_CUDA, "launch_grid_refresh_tail: %s", cudaGetErrorString(et));
    // the packed model's derived occupancy, as gfpp_model_pack builds it: the next gfpp_render_frames marches the new grid
    int *occ = const_cast<int *>(m.occ_bounds);
    k_init_bounds<<<1, 32, 0, st>>>(occ);
    CK(cudaGetLastError());
    CK(launch_occupancy_bounds(bits, C * H3 / 8, H3, occ, st));
    uint32_t *coarse = const_cast<uint32_t *>(m.coarse_bits);
    CKN(cudaMemsetAsync(coarse, 0, (size_t)m.coarse_words * 4, st));
    CK(launch_coarse_occupancy(bits, C, H, coarse, st));
    return GFPP_OK;
}

int gfpp_mark_untrained_grid(const float *poses_c2w, uint32_t n_poses, double fx, double fy, double cx, double cy, double bound,
                             uint32_t cascade, uint32_t grid_size, float *density_grid, void *stream) {
    if (!poses_c2w || !density_grid) return fail(GFPP_ERR_INVALID, "mark_untrained_grid: null pointer%s");
    if (!grid_shape_ok(cascade, grid_size))
        return fail(GFPP_ERR_UNSUPPORTED, "mark_untrained_grid: needs cascade 1..8, grid_size a power of two in 8..512, C*H^3 <= 2^30%s");
    if (n_poses == 0 || !(fx != 0.0) || !(fy != 0.0)) return fail(GFPP_ERR_INVALID, "mark_untrained_grid: no poses or zero focal length%s");
    float scale[8], pad[8];
    cascade_constants(bound, cascade, grid_size, scale, nullptr, pad);
    g_launches = 0;
    CK(launch_mark_untrained(poses_c2w, n_poses, (float)(cx / fx), (float)(cy / fy), scale, pad, cascade, grid_size, density_grid,
                             (cudaStream_t)stream));
    return GFPP_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ (F) torso occupancy grid (torso_grid_kernel.cu; grid_kernels.cu)
namespace {

constexpr uint32_t kTorsoGridMax = 4096;
bool torso_grid_ok(uint32_t H) { return H >= 2 && H <= kTorsoGridMax; }   // the cell placement divides by H - 1

struct TorsoGridWork {
    size_t bias_def, bias_can, tmp, partial, thresh, total;
};

TorsoGridWork torso_grid_work_layout(uint32_t H) {
    TorsoGridWork W;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    W.bias_def = take(64 * 4);
    W.bias_can = take(32 * 4);
    W.tmp = take((size_t)H * H * 4);
    W.partial = take((size_t)torso_dilate_ema_blocks(H) * 8);
    W.thresh = take(4);
    W.total = o;
    return W;
}

// the bias block that opens the refresh's workspace is the query's whole workspace
size_t torso_query_work_bytes() { return torso_grid_work_layout(2).tmp; }

// query arguments of the plain torso field of a packed model, bias vectors in the workspace
TorsoQueryArgs torso_query_args(const ModelHost &m, char *ws, const TorsoGridWork &W) {
    TorsoQueryArgs q;
    memset(&q, 0, sizeof(q));
    q.tor_gm = m.tor_gm; q.tor_tab = m.tor_tab;
    q.w_def0 = m.wd0; q.w_def1 = m.wd1; q.w_def2 = m.wd2; q.w_can0 = m.wc0; q.w_can1 = m.wc1; q.w_can2 = m.wc2;
    q.bias_def = (const float *)(ws + W.bias_def); q.bias_can = (const float *)(ws + W.bias_can);
    q.torso_shrink = m.torso_shrink;
    return q;
}

cudaError_t launch_plain_torso_bias(const ModelHost &m, const float *pose6, const float *code, char *ws, const TorsoGridWork &W,
                                    cudaStream_t st) {
    TorsoArgs t;
    memset(&t, 0, sizeof(t));
    t.n_frames = 1; t.pose6 = pose6;
    return launch_torso_frame_bias(t, m.torso_def0_src, m.torso_can0_src, code, (int)m.torso_code_dim, (float *)(ws + W.bias_def),
                                   (float *)(ws + W.bias_can), st);
}

// the cell query into tmp (the reference's y*H + x layout), then dilation + EMA into density_grid_torso and the mean
int torso_refresh(TorsoQueryArgs q, bool sr, uint32_t H, const float *noise, float decay, float *grid, float *mean_out, float *tmp_grid,
                  char *ws, const TorsoGridWork &W, cudaStream_t st) {
    float *tmp = tmp_grid ? tmp_grid : (float *)(ws + W.tmp);
    q.n = H * H; q.grid_size = H; q.noise = noise;
    q.cell_scale = (float)(1.0 - 1.0 / (double)H); q.hgs = (float)(1.0 / (double)H);   // Python floats of radnerf_torso.py:219-227
    q.alpha = tmp;
    CK(sr ? launch_torso_sr_query(q, st) : launch_torso_query(q, st));
    int nl = 0;
    const cudaError_t e = launch_torso_grid_tail(tmp, H, decay, INFINITY, grid, (double *)(ws + W.partial), mean_out,
                                                 (float *)(ws + W.thresh), &nl, st);
    g_launches += nl;
    if (e != cudaSuccess) return fail(GFPP_ERR_CUDA, "launch_torso_grid_tail: %s", cudaGetErrorString(e));
    return GFPP_OK;
}

}  // namespace

extern "C" {

size_t gfpp_torso_grid_workspace_bytes(uint32_t grid_size) {
    return torso_grid_ok(grid_size) ? torso_grid_work_layout(grid_size).total : 0;
}

size_t gfpp_torso_query_workspace_bytes(void) { return torso_query_work_bytes(); }

int gfpp_torso_query(const gfpp_model *model, const float *xy, uint32_t n, const float *pose6, const float *code, float *alpha,
                     float *color, float *deform, void *workspace, size_t workspace_bytes, void *stream) {
    if (!model || !xy || !pose6 || !alpha || !workspace) return fail(GFPP_ERR_INVALID, "torso_query: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "torso_query: model handle not initialised by gfpp_model_pack%s");
    if (!m.has_torso) return fail(GFPP_ERR_INVALID, "torso_query: the model was packed without a torso (has_torso = 0)%s");
    if ((code == nullptr) != (m.torso_code_dim == 0)) return fail(GFPP_ERR_INVALID, "torso_query: code must be given iff torso_code_dim > 0%s");
    if (n >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "torso_query: n must be < 2^31%s");
    if (workspace_bytes < torso_query_work_bytes()) return fail(GFPP_ERR_WORKSPACE, "torso_query: workspace too small%s");
    const TorsoGridWork W = torso_grid_work_layout(2);   // only its bias block is used
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    g_launches = 0;
    if (n == 0) return GFPP_OK;
    CK(launch_plain_torso_bias(m, pose6, code, ws, W, st));
    TorsoQueryArgs q = torso_query_args(m, ws, W);
    q.n = n; q.xy = xy;
    q.alpha = alpha; q.color = color; q.deform = deform;
    CK(launch_torso_query(q, st));
    return GFPP_OK;
}

int gfpp_torso_grid_update(const gfpp_model *model, const float *pose6, const float *code, const float *noise, float decay,
                           float *density_grid_torso, float *mean_out, float *tmp_grid, void *workspace, size_t workspace_bytes,
                           void *stream) {
    if (!model || !pose6 || !noise || !density_grid_torso || !mean_out || !workspace)
        return fail(GFPP_ERR_INVALID, "torso_grid_update: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "torso_grid_update: model handle not initialised by gfpp_model_pack%s");
    if (!m.has_torso) return fail(GFPP_ERR_INVALID, "torso_grid_update: the model was packed without a torso (has_torso = 0)%s");
    if ((code == nullptr) != (m.torso_code_dim == 0))
        return fail(GFPP_ERR_INVALID, "torso_grid_update: code must be given iff torso_code_dim > 0%s");
    const uint32_t H = m.grid_size;
    if (!torso_grid_ok(H)) return fail(GFPP_ERR_UNSUPPORTED, "torso_grid_update: grid_size must be in 2..4096%s");
    const TorsoGridWork W = torso_grid_work_layout(H);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "torso_grid_update: workspace too small%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    g_launches = 0;
    CK(launch_plain_torso_bias(m, pose6, code, ws, W, st));
    return torso_refresh(torso_query_args(m, ws, W), false, H, noise, decay, density_grid_torso, mean_out, tmp_grid, ws, W, st);
}

int gfpp_torso_sr_grid_update(const gfpp_torso_sr_model *model, const float *lm68, const float *code, const float *noise, float decay,
                              float *density_grid_torso, float *mean_out, float *tmp_grid, void *workspace, size_t workspace_bytes,
                              void *stream) {
    if (!model || !lm68 || !noise || !density_grid_torso || !mean_out || !workspace)
        return fail(GFPP_ERR_INVALID, "torso_sr_grid_update: null pointer%s");
    TorsoSrHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kTorsoSrMagic) return fail(GFPP_ERR_INVALID, "torso_sr_grid_update: model handle not initialised by gfpp_torso_sr_pack%s");
    if ((code == nullptr) != (m.code_dim == 0))
        return fail(GFPP_ERR_INVALID, "torso_sr_grid_update: code must be given iff torso_code_dim > 0%s");
    const uint32_t H = m.grid_size;
    if (!torso_grid_ok(H)) return fail(GFPP_ERR_UNSUPPORTED, "torso_sr_grid_update: grid_size must be in 2..4096%s");
    const TorsoGridWork W = torso_grid_work_layout(H);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "torso_sr_grid_update: workspace too small%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    g_launches = 0;
    CK(launch_torso_sr_frame_bias(lm68, 1, m.def0_src, m.can0_src, code, (int)m.code_dim, m.head_aware, (float *)(ws + W.bias_def),
                                  (float *)(ws + W.bias_can), st));
    TorsoQueryArgs q;
    memset(&q, 0, sizeof(q));
    q.tor_gm = m.tor_gm; q.tor_tab = m.tor_tab;
    q.w_def0 = m.wd0; q.w_def1 = m.wd1; q.w_def2 = m.wd2; q.w_can0 = m.wc0; q.w_can1 = m.wc1; q.w_can2 = m.wc2; q.ha = m.ha;
    q.bias_def = (const float *)(ws + W.bias_def); q.bias_can = (const float *)(ws + W.bias_can);
    q.torso_shrink = m.torso_shrink;
    return torso_refresh(q, true, H, noise, decay, density_grid_torso, mean_out, tmp_grid, ws, W, st);
}

int gfpp_model_set_torso_threshold(gfpp_model *model, float density_thresh_torso) {
    if (!model) return fail(GFPP_ERR_INVALID, "model_set_torso_threshold: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "model_set_torso_threshold: model handle not initialised by gfpp_model_pack%s");
    if (!m.has_torso) return fail(GFPP_ERR_INVALID, "model_set_torso_threshold: the model was packed without a torso (has_torso = 0)%s");
    m.density_thresh_torso = density_thresh_torso;
    memcpy(model, &m, sizeof(m));
    return GFPP_OK;
}

int gfpp_torso_sr_set_threshold(gfpp_torso_sr_model *model, float density_thresh_torso) {
    if (!model) return fail(GFPP_ERR_INVALID, "torso_sr_set_threshold: null pointer%s");
    TorsoSrHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kTorsoSrMagic) return fail(GFPP_ERR_INVALID, "torso_sr_set_threshold: model handle not initialised by gfpp_torso_sr_pack%s");
    m.density_thresh_torso = density_thresh_torso;
    memcpy(model, &m, sizeof(m));
    return GFPP_OK;
}

// ---------------------------------------------------------------- (G) trainable head field
static uint32_t field_ctas(uint32_t M) {
    const uint32_t tiles = (M + FIELD_TP - 1) / FIELD_TP;
    return tiles < (uint32_t)FIELD_CTAS ? tiles : (uint32_t)FIELD_CTAS;
}
static size_t field_wt_bytes() { return (FieldWt::total * 4 + 255) / 256 * 256; }

// Validates the desc (everything the kernels read from it) and fills the model half of FieldArgs; no CUDA call.
static int field_setup(const char *who, const gfpp_model_desc *d, FieldArgs &a) {
    if (!d) return fail(GFPP_ERR_INVALID, "%s: null desc", who);
    memset(&a, 0, sizeof(a));
    const gfpp_grid_desc *gd[2] = {&d->position_grid, &d->ambient_grid};
    GridMeta *gm[2] = {&a.pos_gm, &a.amb_gm};
    for (int i = 0; i < 2; ++i) {
        if (!gd[i]->embeddings || !gd[i]->offsets_host) return fail(GFPP_ERR_INVALID, "%s: null grid table or offsets", who);
        if (gd[i]->num_levels != 16 ||
            fill_grid_meta(*gm[i], gd[i]->offsets_host, gd[i]->input_dim, gd[i]->num_levels, gd[i]->log2_per_level_scale, gd[i]->base_resolution,
                           gd[i]->gridtype, gd[i]->align_corners, gd[i]->interp) != 0)
            return fail(GFPP_ERR_UNSUPPORTED, "%s: grids must have 16 levels x 2 features, 2-D or 3-D", who);
        if (((uintptr_t)gd[i]->embeddings & 7u) != 0) return fail(GFPP_ERR_INVALID, "%s: grid tables must be 8-byte aligned", who);
    }
    if (a.pos_gm.dim != 3) return fail(GFPP_ERR_UNSUPPORTED, "%s: the position grid must be 3-D", who);
    const float *w[8] = {d->ambient_w[0], d->ambient_w[1], d->ambient_w[2], d->sigma_w[0], d->sigma_w[1], d->sigma_w[2], d->color_w[0], d->color_w[1]};
    for (int i = 0; i < 8; ++i) {
        if (!w[i]) return fail(GFPP_ERR_INVALID, "%s: null weight", who);
        if (!aligned16(w[i])) return fail(GFPP_ERR_INVALID, "%s: weights must be 16-byte aligned", who);
        a.w[i] = w[i];
    }
    if (d->cond_dim != 64) return fail(GFPP_ERR_UNSUPPORTED, "%s: cond_dim must be 64", who);
    if (d->ind_dim > 16 || d->ind_dim % 4 != 0) return fail(GFPP_ERR_UNSUPPORTED, "%s: ind_dim must be 0, 4, 8, 12 or 16", who);
    if ((d->ind_dim > 0) != (d->individual_code != nullptr)) return fail(GFPP_ERR_INVALID, "%s: individual_code must be given iff ind_dim > 0", who);
    if (d->mlp_precision != 0) return fail(GFPP_ERR_UNSUPPORTED, "%s: the training field runs in fp32 only (mlp_precision 0)", who);
    a.pos_tab = (const float2 *)d->position_grid.embeddings;
    a.amb_tab = (const float2 *)d->ambient_grid.embeddings;
    a.code = d->individual_code;
    a.ind_dim = (int)d->ind_dim;
    a.amb_dim = (int)a.amb_gm.dim;
    a.bound = d->bound;
    return GFPP_OK;
}

size_t gfpp_field_backward_workspace_bytes(uint32_t M) {
    if (M >= (1u << 30)) return 0;
    return field_wt_bytes() + (size_t)field_ctas(M) * FieldPart::total * 4;
}

int gfpp_field_forward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat, float *sigma,
                       float *color, float *ambient_pos, void *workspace, size_t workspace_bytes, void *stream) {
    FieldArgs a;
    const int rc = field_setup("field_forward", desc, a);
    if (rc != GFPP_OK) return rc;
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    if (!xyzs || !dirs || !cond_feat || !sigma || !color || !ambient_pos || !workspace) return fail(GFPP_ERR_INVALID, "field_forward: null pointer%s");
    if (M >= (1u << 30)) return fail(GFPP_ERR_UNSUPPORTED, "field_forward: M must be < 2^30%s");
    if (workspace_bytes < field_wt_bytes()) return fail(GFPP_ERR_WORKSPACE, "field_forward: workspace too small%s");
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "field_forward: workspace must be 256-byte aligned%s");
    a.M = M; a.xyzs = xyzs; a.dirs = dirs; a.cond = cond_feat;
    a.wt = (float *)workspace;
    a.sigma = sigma; a.color = color; a.ambient = ambient_pos;
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_field_relayout(a, st));
    CK(launch_field_fwd(a, st));
    return GFPP_OK;
}

int gfpp_field_backward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat,
                        const float *grad_sigma, const float *grad_color, const float *grad_ambient_pos, float *const grad_w[8], float *grad_cond,
                        float *grad_code, float *grad_position_table, float *grad_ambient_table, void *workspace, size_t workspace_bytes,
                        void *stream) {
    FieldArgs a;
    const int rc = field_setup("field_backward", desc, a);
    if (rc != GFPP_OK) return rc;
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    if (!xyzs || !dirs || !cond_feat || !grad_sigma || !grad_color || !grad_ambient_pos || !grad_w || !grad_cond || !grad_position_table ||
        !grad_ambient_table || !workspace || (a.ind_dim > 0 && !grad_code))
        return fail(GFPP_ERR_INVALID, "field_backward: null pointer%s");
    for (int i = 0; i < 8; ++i)
        if (!grad_w[i]) return fail(GFPP_ERR_INVALID, "field_backward: null weight gradient%s");
    if (((uintptr_t)grad_position_table & 7u) || ((uintptr_t)grad_ambient_table & 7u))
        return fail(GFPP_ERR_INVALID, "field_backward: table gradients must be 8-byte aligned%s");
    if (M >= (1u << 30)) return fail(GFPP_ERR_UNSUPPORTED, "field_backward: M must be < 2^30%s");
    if (workspace_bytes < gfpp_field_backward_workspace_bytes(M)) return fail(GFPP_ERR_WORKSPACE, "field_backward: workspace too small%s");
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "field_backward: workspace must be 256-byte aligned%s");
    a.M = M; a.xyzs = xyzs; a.dirs = dirs; a.cond = cond_feat;
    a.wt = (float *)workspace;
    a.part = (float *)((char *)workspace + field_wt_bytes());
    a.n_cta = field_ctas(M);
    a.g_sigma = grad_sigma; a.g_color = grad_color; a.g_ambient = grad_ambient_pos;
    a.g_pos_tab = (float2 *)grad_position_table; a.g_amb_tab = (float2 *)grad_ambient_table;
    for (int i = 0; i < 8; ++i) a.g_w[i] = grad_w[i];
    a.g_cond = grad_cond; a.g_code = grad_code;
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_field_relayout(a, st));
    CK(launch_field_bwd(a, st));
    CK(launch_field_reduce(a, st));
    return GFPP_OK;
}

// ---------------------------------------------------------------- (H) and (I) trainable torso fields
// Both fields run the kernels of torso_train_kernel.cu: SR = false for the plain torso (H), SR = true for the torso-SR model (I).
extern "C++" {   // the helpers are templates
static uint32_t torso_field_ctas(uint32_t M) {
    const uint32_t tiles = (M + TORSO_TRAIN_TP - 1) / TORSO_TRAIN_TP;
    return tiles < (uint32_t)TORSO_TRAIN_CTAS ? tiles : (uint32_t)TORSO_TRAIN_CTAS;
}
template <bool SR> static size_t torso_wt_bytes() { return (TorsoWt<SR>::total * 4 + 255) / 256 * 256; }
template <bool SR> static size_t torso_field_ws_bytes(uint32_t M) {
    if (M >= (1u << 31)) return 0;
    return torso_wt_bytes<SR>() + (size_t)torso_field_ctas(M) * TorsoPart<SR>::total * 4;
}

// Validates what both fields' descs hold -- the torso grid, the six weights, torso_code_dim -- and the code, and fills that part of
// TorsoTrainArgs; no CUDA call.  Desc is gfpp_model_desc (H) or gfpp_torso_sr_desc (I).
template <class Desc> static int torso_field_setup(const char *who, const Desc *d, const float *code, TorsoTrainArgs &a) {
    if (!d) return fail(GFPP_ERR_INVALID, "%s: null desc", who);
    memset(&a, 0, sizeof(a));
    const gfpp_grid_desc &g = d->torso_grid;
    if (!g.embeddings || !g.offsets_host) return fail(GFPP_ERR_INVALID, "%s: null torso grid table or offsets", who);
    if (g.num_levels != 16 ||
        fill_grid_meta(a.gm, g.offsets_host, g.input_dim, g.num_levels, g.log2_per_level_scale, g.base_resolution, g.gridtype,
                       g.align_corners, g.interp) != 0 || a.gm.dim != 2)
        return fail(GFPP_ERR_UNSUPPORTED, "%s: the torso grid must be 2-D with 16 levels x 2 features", who);
    if (((uintptr_t)g.embeddings & 7u) != 0) return fail(GFPP_ERR_INVALID, "%s: the torso grid table must be 8-byte aligned", who);
    for (int i = 0; i < 3; ++i) {
        if (!d->torso_deform_w[i] || !d->torso_canon_w[i]) return fail(GFPP_ERR_INVALID, "%s: null torso weight", who);
        a.w_def[i] = d->torso_deform_w[i];
        a.w_can[i] = d->torso_canon_w[i];
    }
    if (d->torso_code_dim > 10) return fail(GFPP_ERR_UNSUPPORTED, "%s: torso_code_dim must be <= 10", who);
    if ((code == nullptr) != (d->torso_code_dim == 0)) return fail(GFPP_ERR_INVALID, "%s: code must be given iff torso_code_dim > 0", who);
    a.tab = (const float2 *)g.embeddings;
    a.code = code;
    a.code_dim = (int)d->torso_code_dim;
    a.shrink = d->torso_shrink;
    return GFPP_OK;
}

// The section (I) setup: the shared part, then lm68, the head-aware encoder and its image / weights_sum inputs.
static int torso_sr_field_setup(const char *who, const gfpp_torso_sr_desc *d, const float *lm68, const float *code, const float *image,
                                const float *weights_sum, TorsoTrainArgs &a) {
    const int rc = torso_field_setup(who, d, code, a);
    if (rc != GFPP_OK) return rc;
    if (!lm68) return fail(GFPP_ERR_INVALID, "%s: null lm68", who);
    if ((image == nullptr) != (weights_sum == nullptr)) return fail(GFPP_ERR_INVALID, "%s: image and weights_sum must both be given or both be NULL", who);
    if (d->head_aware) {
        for (int i = 0; i < 3; ++i) {
            if (!d->ha_w[i] || !d->ha_b[i]) return fail(GFPP_ERR_INVALID, "%s: null head-aware encoder weight", who);
            a.ha_w[i] = d->ha_w[i];
            a.ha_b[i] = d->ha_b[i];
        }
    } else if (image) {
        return fail(GFPP_ERR_INVALID, "%s: image and weights_sum are only read with head_aware", who);
    }
    a.head_aware = d->head_aware ? 1 : 0;
    a.cond = lm68;
    a.image = image;
    a.wsum = weights_sum;
    return GFPP_OK;
}

// The forward's checks after the setup, then the relayout into the workspace; M = 0 returns before it.
template <bool SR>
static int torso_field_relayout(const char *who, TorsoTrainArgs &a, const float *xy, uint32_t M, const float *alpha, const float *color,
                                const float *deform, void *workspace, size_t workspace_bytes, cudaStream_t st) {
    if (!xy || !alpha || !color || !deform || !workspace) return fail(GFPP_ERR_INVALID, "%s: null pointer", who);
    if (M >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "%s: M must be < 2^31", who);
    if (workspace_bytes < torso_wt_bytes<SR>()) return fail(GFPP_ERR_WORKSPACE, "%s: workspace too small", who);
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "%s: workspace must be 256-byte aligned", who);
    a.wt = (float *)workspace;
    CK(launch_torso_field_relayout<SR>(a, st));
    return GFPP_OK;
}

// The backward after the setup: the checks both fields share, then relayout, backward and reduce.
template <bool SR>
static int torso_field_backward(const char *who, TorsoTrainArgs &a, const float *xy, uint32_t M, const float *grad_alpha,
                                const float *grad_color, const float *grad_deform, float *const grad_deform_w[3],
                                float *const grad_canon_w[3], float *grad_code, float *grad_torso_table, void *workspace,
                                size_t workspace_bytes, void *stream) {
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    if (!xy || !grad_alpha || !grad_color || !grad_deform || !grad_deform_w || !grad_canon_w || !grad_torso_table || !workspace ||
        (a.code_dim > 0 && !grad_code))
        return fail(GFPP_ERR_INVALID, "%s: null pointer", who);
    for (int i = 0; i < 3; ++i)
        if (!grad_deform_w[i] || !grad_canon_w[i]) return fail(GFPP_ERR_INVALID, "%s: null weight gradient", who);
    if (((uintptr_t)grad_torso_table & 7u) != 0) return fail(GFPP_ERR_INVALID, "%s: the table gradient must be 8-byte aligned", who);
    if (M >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "%s: M must be < 2^31", who);
    if (workspace_bytes < torso_field_ws_bytes<SR>(M)) return fail(GFPP_ERR_WORKSPACE, "%s: workspace too small", who);
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "%s: workspace must be 256-byte aligned", who);
    a.M = M; a.xy = xy;
    a.wt = (float *)workspace;
    a.part = (float *)((char *)workspace + torso_wt_bytes<SR>());
    a.n_cta = torso_field_ctas(M);
    a.g_alpha = grad_alpha; a.g_color = grad_color; a.g_deform = grad_deform;
    a.g_tab = (float2 *)grad_torso_table;
    for (int i = 0; i < 3; ++i) { a.g_def[i] = grad_deform_w[i]; a.g_can[i] = grad_canon_w[i]; }
    a.g_code = grad_code;
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_torso_field_relayout<SR>(a, st));
    CK(launch_torso_field_bwd<SR>(a, st));
    CK(launch_torso_field_reduce<SR>(a, st));
    return GFPP_OK;
}

}  // extern "C++"

size_t gfpp_torso_field_workspace_bytes(uint32_t M) { return torso_field_ws_bytes<false>(M); }

int gfpp_torso_field_forward(const gfpp_model_desc *desc, const float *xy, uint32_t M, const float *pose6, const float *code, float *alpha,
                             float *color, float *deform, void *workspace, size_t workspace_bytes, void *stream) {
    TorsoTrainArgs a;
    int rc = torso_field_setup("torso_field_forward", desc, code, a);
    if (rc != GFPP_OK) return rc;
    if (!pose6) return fail(GFPP_ERR_INVALID, "torso_field_forward: null pose6%s");
    a.cond = pose6;
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    cudaStream_t st = (cudaStream_t)stream;
    rc = torso_field_relayout<false>("torso_field_forward", a, xy, M, alpha, color, deform, workspace, workspace_bytes, st);
    if (rc != GFPP_OK) return rc;
    // the inference query's kernel on the re-laid-out weights: the same values as gfpp_torso_query at the same parameters
    using W = TorsoWt<false>;
    TorsoQueryArgs q;
    memset(&q, 0, sizeof(q));
    q.tor_gm = a.gm; q.tor_tab = a.tab;
    q.w_def0 = a.wt + W::wd0; q.w_def1 = a.wt + W::wd1; q.w_def2 = a.wt + W::wd2;
    q.w_can0 = a.wt + W::wc0; q.w_can1 = a.wt + W::wc1; q.w_can2 = a.wt + W::wc2;
    q.bias_def = a.wt + W::bias_def; q.bias_can = a.wt + W::bias_can;
    q.torso_shrink = a.shrink;
    q.n = M; q.xy = xy;
    q.alpha = alpha; q.color = color; q.deform = deform;
    CK(launch_torso_query(q, st));
    return GFPP_OK;
}

int gfpp_torso_field_backward(const gfpp_model_desc *desc, const float *xy, uint32_t M, const float *pose6, const float *code,
                              const float *grad_alpha, const float *grad_color, const float *grad_deform, float *const grad_deform_w[3],
                              float *const grad_canon_w[3], float *grad_code, float *grad_torso_table, void *workspace, size_t workspace_bytes,
                              void *stream) {
    TorsoTrainArgs a;
    const int rc = torso_field_setup("torso_field_backward", desc, code, a);
    if (rc != GFPP_OK) return rc;
    if (!pose6) return fail(GFPP_ERR_INVALID, "torso_field_backward: null pose6%s");
    a.cond = pose6;
    return torso_field_backward<false>("torso_field_backward", a, xy, M, grad_alpha, grad_color, grad_deform, grad_deform_w, grad_canon_w,
                                       grad_code, grad_torso_table, workspace, workspace_bytes, stream);
}

size_t gfpp_torso_sr_field_workspace_bytes(uint32_t M) { return torso_field_ws_bytes<true>(M); }

int gfpp_torso_sr_field_forward(const gfpp_torso_sr_desc *desc, const float *xy, uint32_t M, const float *lm68, const float *code,
                                const float *image, const float *weights_sum, float *alpha, float *color, float *deform, void *workspace,
                                size_t workspace_bytes, void *stream) {
    TorsoTrainArgs a;
    int rc = torso_sr_field_setup("torso_sr_field_forward", desc, lm68, code, image, weights_sum, a);
    if (rc != GFPP_OK) return rc;
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    cudaStream_t st = (cudaStream_t)stream;
    rc = torso_field_relayout<true>("torso_sr_field_forward", a, xy, M, alpha, color, deform, workspace, workspace_bytes, st);
    if (rc != GFPP_OK) return rc;
    // k_torso_sr's field in its point mode on the re-laid-out weights: the same values as the render epilogue at the same parameters
    using W = TorsoWt<true>;
    TorsoSrArgs t;
    memset(&t, 0, sizeof(t));
    t.tor_gm = a.gm; t.tor_tab = a.tab;
    t.w_def0 = a.wt + W::wd0; t.w_def1 = a.wt + W::wd1; t.w_def2 = a.wt + W::wd2;
    t.w_can0 = a.wt + W::wc0; t.w_can1 = a.wt + W::wc1; t.w_can2 = a.wt + W::wc2;
    t.ha = a.head_aware ? a.wt + W::ha : nullptr;
    t.bias_def = a.wt + W::bias_def; t.bias_can = a.wt + W::bias_can;
    t.torso_shrink = a.shrink;
    t.bg_coords = xy;
    t.n_frames = 1; t.n_rays = (int)M;
    t.image = image; t.wsum = weights_sum;
    t.torso_alpha = alpha; t.torso_rgb = color; t.deform = deform;
    CK(launch_torso_sr_points(t, st));
    return GFPP_OK;
}

int gfpp_torso_sr_field_backward(const gfpp_torso_sr_desc *desc, const float *xy, uint32_t M, const float *lm68, const float *code,
                                 const float *image, const float *weights_sum, const float *grad_alpha, const float *grad_color,
                                 const float *grad_deform, float *const grad_deform_w[3], float *const grad_canon_w[3],
                                 float *const grad_ha_w[3], float *const grad_ha_b[3], float *grad_code, float *grad_torso_table,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    TorsoTrainArgs a;
    const int rc = torso_sr_field_setup("torso_sr_field_backward", desc, lm68, code, image, weights_sum, a);
    if (rc != GFPP_OK) return rc;
    if ((grad_ha_w == nullptr) != (a.head_aware == 0) || (grad_ha_b == nullptr) != (a.head_aware == 0))
        return fail(GFPP_ERR_INVALID, "torso_sr_field_backward: grad_ha_w / grad_ha_b must be given iff head_aware%s");
    if (a.head_aware)
        for (int i = 0; i < 3; ++i) {
            if (!grad_ha_w[i] || !grad_ha_b[i]) return fail(GFPP_ERR_INVALID, "torso_sr_field_backward: null head-aware gradient%s");
            a.g_ha_w[i] = grad_ha_w[i];
            a.g_ha_b[i] = grad_ha_b[i];
        }
    return torso_field_backward<true>("torso_sr_field_backward", a, xy, M, grad_alpha, grad_color, grad_deform, grad_deform_w, grad_canon_w,
                                      grad_code, grad_torso_table, workspace, workspace_bytes, stream);
}

// ---------------------------------------------------------------- (J) trainable head field on tensor cores
static uint32_t field_tc_ctas(uint32_t M) {
    const uint32_t tiles = (M + FIELD_TC_TP - 1) / FIELD_TC_TP;
    return tiles < (uint32_t)FIELD_CTAS ? tiles : (uint32_t)FIELD_CTAS;
}

size_t gfpp_field_tc_workspace_bytes(uint32_t M) {
    if (M >= (1u << 30)) return 0;
    return (size_t)FieldTcImg::total + (size_t)field_tc_ctas(M) * FieldPart::total * 4;
}

int gfpp_field_tc_forward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat, float *sigma,
                          float *color, float *ambient_pos, void *workspace, size_t workspace_bytes, void *stream) {
    FieldTcArgs t;
    FieldArgs &a = t.f;
    const int rc = field_setup("field_tc_forward", desc, a);
    if (rc != GFPP_OK) return rc;
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    if (!xyzs || !dirs || !cond_feat || !sigma || !color || !ambient_pos || !workspace) return fail(GFPP_ERR_INVALID, "field_tc_forward: null pointer%s");
    if (M >= (1u << 30)) return fail(GFPP_ERR_UNSUPPORTED, "field_tc_forward: M must be < 2^30%s");
    if (workspace_bytes < FieldTcImg::total) return fail(GFPP_ERR_WORKSPACE, "field_tc_forward: workspace too small%s");
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "field_tc_forward: workspace must be 256-byte aligned%s");
    a.M = M; a.xyzs = xyzs; a.dirs = dirs; a.cond = cond_feat;
    t.img = (unsigned char *)workspace;
    a.wt = (float *)(t.img + FieldTcImg::bias);
    a.sigma = sigma; a.color = color; a.ambient = ambient_pos;
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_field_tc_relayout(t, st));
    CK(launch_field_tc_fwd(t, st));
    return GFPP_OK;
}

int gfpp_field_tc_backward(const gfpp_model_desc *desc, const float *xyzs, const float *dirs, uint32_t M, const float *cond_feat,
                           const float *grad_sigma, const float *grad_color, const float *grad_ambient_pos, float *const grad_w[8], float *grad_cond,
                           float *grad_code, float *grad_position_table, float *grad_ambient_table, void *workspace, size_t workspace_bytes,
                           void *stream) {
    FieldTcArgs t;
    FieldArgs &a = t.f;
    const int rc = field_setup("field_tc_backward", desc, a);
    if (rc != GFPP_OK) return rc;
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    if (!xyzs || !dirs || !cond_feat || !grad_sigma || !grad_color || !grad_ambient_pos || !grad_w || !grad_cond || !grad_position_table ||
        !grad_ambient_table || !workspace || (a.ind_dim > 0 && !grad_code))
        return fail(GFPP_ERR_INVALID, "field_tc_backward: null pointer%s");
    for (int i = 0; i < 8; ++i)
        if (!grad_w[i]) return fail(GFPP_ERR_INVALID, "field_tc_backward: null weight gradient%s");
    if (((uintptr_t)grad_position_table & 7u) || ((uintptr_t)grad_ambient_table & 7u))
        return fail(GFPP_ERR_INVALID, "field_tc_backward: table gradients must be 8-byte aligned%s");
    if (M >= (1u << 30)) return fail(GFPP_ERR_UNSUPPORTED, "field_tc_backward: M must be < 2^30%s");
    if (workspace_bytes < gfpp_field_tc_workspace_bytes(M)) return fail(GFPP_ERR_WORKSPACE, "field_tc_backward: workspace too small%s");
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "field_tc_backward: workspace must be 256-byte aligned%s");
    a.M = M; a.xyzs = xyzs; a.dirs = dirs; a.cond = cond_feat;
    t.img = (unsigned char *)workspace;
    a.wt = (float *)(t.img + FieldTcImg::bias);
    a.part = (float *)(t.img + FieldTcImg::total);
    a.n_cta = field_tc_ctas(M);
    a.g_sigma = grad_sigma; a.g_color = grad_color; a.g_ambient = grad_ambient_pos;
    a.g_pos_tab = (float2 *)grad_position_table; a.g_amb_tab = (float2 *)grad_ambient_table;
    for (int i = 0; i < 8; ++i) a.g_w[i] = grad_w[i];
    a.g_cond = grad_cond; a.g_code = grad_code;
    cudaStream_t st = (cudaStream_t)stream;
    CK(launch_field_tc_relayout(t, st));
    CK(launch_field_tc_bwd(t, st));
    CK(launch_field_reduce(a, st));
    return GFPP_OK;
}

}  // extern "C"

// ---------------------------------------------------------------- (K) frozen head of the torso training steps
namespace {
struct FrozenWork { size_t narrow, depth, rays_t, survivors, hits, zero_begin, hist, counters, zero_end, cond, total; };
FrozenWork frozen_work_layout(uint32_t N, uint32_t max_steps) {
    FrozenWork W;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) / 256 * 256; return r; };
    W.narrow = take(8 * 128 * 4);          // the packed narrow rows with this call's individual code folded into row 7
    W.depth = take((size_t)N * 4);
    W.rays_t = take((size_t)N * 4);
    W.survivors = take((size_t)N * 4);
    W.hits = take((size_t)N * 64);         // HitRecord (head_common.cuh)
    W.zero_begin = o;
    W.hist = take((size_t)(max_steps + 2) * 4);
    W.counters = take(16 * 4);
    W.zero_end = o;
    W.cond = take(64 * 2 * 2);             // fp16 hi + lo images of cond_feat (v2 head kernel)
    W.total = o;
    return W;
}
}  // namespace

extern "C" {

size_t gfpp_frozen_head_workspace_bytes(uint32_t N, uint32_t max_steps) {
    if (N == 0 || N >= (1u << 31) || max_steps < 1 || max_steps > 4096) return 0;
    return frozen_work_layout(N, max_steps).total;
}

int gfpp_frozen_head(const gfpp_model *model, const float *rays_o, const float *rays_d, uint32_t N, const float aabb[6], const float *cond_feat,
                     const float *code, const float *noises, float dt_gamma, uint32_t max_steps, float T_thresh, float *weights_sum, float *image,
                     void *workspace, size_t workspace_bytes, void *stream) {
    if (!model || !rays_o || !rays_d || !aabb || !cond_feat || !weights_sum || !image || !workspace)
        return fail(GFPP_ERR_INVALID, "frozen_head: null pointer%s");
    ModelHost m;
    memcpy(&m, model, sizeof(m));
    if (m.magic != kMagic) return fail(GFPP_ERR_INVALID, "frozen_head: model handle not initialised by gfpp_model_pack%s");
    if (N == 0) return fail(GFPP_ERR_INVALID, "frozen_head: no rays%s");
    if (N >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "frozen_head: N must be < 2^31%s");
    if (max_steps < 1 || max_steps > 4096) return fail(GFPP_ERR_UNSUPPORTED, "frozen_head: max_steps must be in 1..4096%s");
    if ((m.ind_dim > 0) != (code != nullptr)) return fail(GFPP_ERR_INVALID, "frozen_head: code must be given iff the model has individual codes%s");
    for (int k = 0; k < 3; ++k)
        if (!(aabb[k] <= aabb[3 + k])) return fail(GFPP_ERR_INVALID, "frozen_head: aabb must be (xmin, ymin, zmin, xmax, ymax, zmax)%s");
    const bool use_v2 = m.v2_ok && (m.mlp_precision == 4 || (m.mlp_precision == 1 && getenv("GFPP_HEAD_V1") == nullptr));
    if (m.mlp_precision == 4 && !use_v2) return fail(GFPP_ERR_UNSUPPORTED, "frozen_head: robust mode unavailable for this model%s");
    const FrozenWork W = frozen_work_layout(N, max_steps);
    if (workspace_bytes < W.total) return fail(GFPP_ERR_WORKSPACE, "frozen_head: workspace too small%s");
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "frozen_head: workspace must be 256-byte aligned%s");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    g_launches = 0;
    CKN(cudaMemsetAsync(ws + W.zero_begin, 0, W.zero_end - W.zero_begin, st));
    // this call's individual code: a copy of the packed narrow rows with `code` folded into the colour-L0 bias (row 7) exactly as
    // gfpp_model_pack folds row 0; the packed model is never written, so render() keeps using row 0
    float *narrow = (float *)(ws + W.narrow);
    CKN(cudaMemcpyAsync(narrow, m.narrow, (code ? 7 : 8) * 128 * 4, cudaMemcpyDeviceToDevice, st));
    if (code) CK(launch_fold_bias(m.color0_src, 16 + 128 + m.ind_dim, 144, m.ind_dim, code, 128, narrow + 7 * 128, st));

    HeadArgs a;
    memset(&a, 0, sizeof(a));
    a.pos_gm = m.pos_gm; a.amb_gm = m.amb_gm;
    a.pos_tab = m.pos_tab; a.amb_tab = m.amb_tab;
    a.pos_quads = m.pos_quads; a.amb_quads = m.amb_quads;
    a.pos_octs = m.pos_octs; a.amb_octs = m.amb_octs;
    a.wide = m.wide; a.narrow = narrow;
    for (int c = 0; c < HEAD_NCHUNK; ++c) { a.chunk_off[c] = m.chunk_off[c]; a.chunk_k[c] = kChunkK[c]; }
    march_const_init(a.mc, m.bound, dt_gamma, max_steps, m.cascade, m.grid_size, m.bitfield);
    a.occ_bounds = m.occ_bounds;
    a.coarse_bits = m.coarse_bits;
    a.coarse_words = m.coarse_words;
    memcpy(a.aabb, aabb, sizeof(a.aabb));
    a.min_near = m.min_near; a.density_scale = m.density_scale;
    // the occupied-box shortcut assumes no sample position is clamped to the cube: it holds for this call's aabb only if it lies inside
    const float cube = m.bound;
    a.use_occ_box = (m.cascade == 1 && aabb[0] >= -cube && aabb[1] >= -cube && aabb[2] >= -cube && aabb[3] <= cube && aabb[4] <= cube &&
                     aabb[5] <= cube) ? 1 : 0;
    a.n_frames = 1; a.n_rays = (int)N;
    a.rays_o = rays_o; a.rays_d = rays_d;
    a.cond_feat = cond_feat;
    a.max_steps = (int)max_steps; a.T_thresh = T_thresh;
    a.noises = noises;
    a.image = image;
    a.wsum = weights_sum;
    a.depth = (float *)(ws + W.depth);
    a.rays_t = (float *)(ws + W.rays_t);
    a.hist = (int *)(ws + W.hist);
    a.survivors = (int *)(ws + W.survivors);
    int *counters = (int *)(ws + W.counters);
    a.n_survivors = counters + 2;
    a.hits = (uint4 *)(ws + W.hits);
    a.n_hits = counters + 3;
    a.pass = 1;
    a.cursor = counters + 0;
    // pass 1 only: a ray that reaches max_steps samples is final (march_rays_train gives it no more), so there is no schedule,
    // no pass 2 and no epilogue
    CK(launch_ray_setup(a, st));
    if (m.mlp_precision == 0) CK(launch_head(a, -1, st, true));
    else if (use_v2) {
        HeadV2Args v2;
        v2.w_stream = m.v2_stream; v2.w_res = m.v2_res; v2.pos_step = m.v2_pos_step;
        v2.cond_hi = (const unsigned char *)(ws + W.cond);
        v2.cond_lo = v2.cond_hi + 128;
        CK(launch_cond_images(cond_feat, 1, ws + W.cond, ws + W.cond + 128, st));
        CK(launch_head_v2(a, v2, m.mlp_precision, st, true));
    } else CK(launch_head_tc(a, m.tc, m.mlp_precision, -1, st, true));
    return GFPP_OK;
}

}  // extern "C"

// ---------------------------------------------------------------- (M) torso pass of the torso training steps
extern "C" {

size_t gfpp_torso_pass_workspace_bytes(uint32_t N) {
    if (N == 0 || N >= (1u << 31)) return 0;
    return ((size_t)torso_mask_tiles(N) * 4 + 255) / 256 * 256;
}

int gfpp_torso_mask(const float *density_grid_torso, uint32_t G, float thr, const float *bg_coords, uint32_t N, const float *image,
                    const float *weights_sum, int32_t *idx, int32_t *slot, float *xy, float *image_m, float *weights_sum_m, int32_t *count,
                    void *workspace, size_t workspace_bytes, void *stream) {
    if (!density_grid_torso || !bg_coords || !idx || !slot || !xy || !count || !workspace) return fail(GFPP_ERR_INVALID, "torso_mask: null pointer%s");
    if ((image == nullptr) != (weights_sum == nullptr) || (image == nullptr) != (image_m == nullptr) || (image == nullptr) != (weights_sum_m == nullptr))
        return fail(GFPP_ERR_INVALID, "torso_mask: image, weights_sum and their gathers must all be given or all be NULL%s");
    if (N == 0) return fail(GFPP_ERR_INVALID, "torso_mask: no pixels%s");
    if (N >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "torso_mask: N must be < 2^31%s");
    if (G < 2 || G > 4096) return fail(GFPP_ERR_UNSUPPORTED, "torso_mask: grid_size must be in 2..4096%s");
    if ((((uintptr_t)bg_coords | (uintptr_t)xy) & 7u) != 0) return fail(GFPP_ERR_INVALID, "torso_mask: bg_coords and xy must be 8-byte aligned%s");
    if (workspace_bytes < gfpp_torso_pass_workspace_bytes(N)) return fail(GFPP_ERR_WORKSPACE, "torso_mask: workspace too small%s");
    if (((uintptr_t)workspace & 255u) != 0) return fail(GFPP_ERR_INVALID, "torso_mask: workspace must be 256-byte aligned%s");
    g_launches = 0;
    CK(launch_torso_mask(density_grid_torso, G, thr, bg_coords, image, weights_sum, N, idx, slot, xy, image_m, weights_sum_m, count,
                         (int *)workspace, (cudaStream_t)stream));
    g_launches = 3;
    return GFPP_OK;
}

// the checks the composite's two directions share; no CUDA call
static int torso_composite_check(const char *who, uint32_t N, uint32_t M, const float *alpha, const float *color, const float *image,
                                 const float *weights_sum, const float *bg_color, uint32_t bg_mode) {
    if (!image || !weights_sum) return fail(GFPP_ERR_INVALID, "%s: null pointer", who);
    if (M > 0 && (!alpha || !color)) return fail(GFPP_ERR_INVALID, "%s: alpha and color must be given when M > 0", who);
    if (N == 0) return fail(GFPP_ERR_INVALID, "%s: no pixels", who);
    if (N >= (1u << 31)) return fail(GFPP_ERR_UNSUPPORTED, "%s: N must be < 2^31", who);
    if (M > N) return fail(GFPP_ERR_INVALID, "%s: more masked points than pixels", who);
    if (bg_mode > 2) return fail(GFPP_ERR_INVALID, "%s: bg_mode must be 0 (scalar 1), 1 (one colour) or 2 (per pixel)", who);
    if ((bg_color == nullptr) != (bg_mode == 0)) return fail(GFPP_ERR_INVALID, "%s: bg_color must be given iff bg_mode > 0", who);
    return GFPP_OK;
}

int gfpp_torso_composite_forward(const int32_t *slot, uint32_t N, uint32_t M, const float *alpha, const float *color, const float *image,
                                 const float *weights_sum, const float *bg_color, uint32_t bg_mode, float *torso_alpha_map,
                                 float *torso_rgb_map, float *rgb_map, void *stream) {
    if (!slot || !torso_alpha_map || !torso_rgb_map || !rgb_map) return fail(GFPP_ERR_INVALID, "torso_composite_forward: null pointer%s");
    const int rc = torso_composite_check("torso_composite_forward", N, M, alpha, color, image, weights_sum, bg_color, bg_mode);
    if (rc != GFPP_OK) return rc;
    g_launches = 0;
    CK(launch_torso_composite_fwd(slot, N, alpha, color, image, weights_sum, bg_color, bg_mode, torso_alpha_map, torso_rgb_map, rgb_map,
                                  (cudaStream_t)stream));
    return GFPP_OK;
}

int gfpp_torso_composite_backward(const int32_t *idx, uint32_t N, uint32_t M, const float *alpha, const float *color, const float *image,
                                  const float *weights_sum, const float *bg_color, uint32_t bg_mode, const float *grad_torso_alpha_map,
                                  const float *grad_torso_rgb_map, const float *grad_rgb_map, float *grad_alpha, float *grad_color,
                                  void *stream) {
    const int rc = torso_composite_check("torso_composite_backward", N, M, alpha, color, image, weights_sum, bg_color, bg_mode);
    if (rc != GFPP_OK) return rc;
    if (M > 0 && (!idx || !grad_alpha || !grad_color)) return fail(GFPP_ERR_INVALID, "torso_composite_backward: null pointer%s");
    g_launches = 0;
    if (M == 0) return GFPP_OK;
    CK(launch_torso_composite_bwd(idx, M, alpha, color, image, weights_sum, bg_color, bg_mode, grad_torso_alpha_map, grad_torso_rgb_map,
                                  grad_rgb_map, grad_alpha, grad_color, (cudaStream_t)stream));
    return GFPP_OK;
}

}  // extern "C"
