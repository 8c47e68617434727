// torso_pass_kernels.cu -- the per-pixel part of the torso training steps (include/gfpp.h section M), sm_90a.
//
// Between the frozen head (section K) and the torso fields (sections H and I) the reference's torso steps (radnerf_torso.py:165-193,
// radnerf_torso_sr.py:196-221) run, per pixel: the grid_sample mask of density_grid_torso, the boolean-index gathers of bg_coords
// (and, for the SR field's head-aware inputs, of image and weights_sum), the index_put scatters of the field's outputs and the
// three-way composite with its clamp; and the autograd backward of all of that.  Here:
//   * mask + stable compaction: block counts, a one-CTA scan of the counts, a tile-local scan that writes slot / idx and the
//     gathers.  Masked pixels keep their ascending order (the order of bg_coords[mask]); no atomics; M is written on the device.
//   * composite forward: one thread per pixel, the field's outputs read through slot, PyTorch's op order in round-to-nearest
//     intrinsics (no FMA contraction), so the maps are bit-identical to the composed recipe.
//   * composite backward: one thread per masked point, through idx; the clamp's gradient recomputed from the forward's arithmetic.
// The kernels take plain arrays only (no model descriptor): one set serves both torso models.
#include "common.cuh"
#include "launch.cuh"
#include "ops.cuh"
#include "torso_common.cuh"

namespace gfpp {

namespace {

constexpr int MASK_NT = 1024, MASK_ITEMS = 4, MASK_TILE = MASK_NT * MASK_ITEMS;

// occ = grid_sample(density_grid_torso, (x, y)) > thr, in the arithmetic of ATen's CUDA kernel
__device__ __forceinline__ int torso_flag(const float *__restrict__ grid, int G, float thr, const float2 *__restrict__ xy, uint32_t i) {
    const float2 p = xy[i];
    return torsoc::sample_density<true>(grid, G, p.x, p.y) > thr ? 1 : 0;
}

// pass 1: the mask of each tile's pixels into slot (0 / 1), the tile's count into tile_sums
__global__ void __launch_bounds__(MASK_NT) k_torso_mask_count(const float *__restrict__ grid, int G, float thr, const float2 *__restrict__ xy,
                                                              uint32_t N, int32_t *__restrict__ slot, int *__restrict__ tile_sums) {
    __shared__ int sw[65];
    const uint32_t base = blockIdx.x * MASK_TILE + threadIdx.x * MASK_ITEMS;
    int s = 0;
#pragma unroll
    for (int i = 0; i < MASK_ITEMS; ++i)
        if (base + i < N) {
            const int f = torso_flag(grid, G, thr, xy, base + i);
            slot[base + i] = f;
            s += f;
        }
    int total;
    (void)block_exclusive_scan(s, sw, total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// pass 2 (one CTA): exclusive scan of the tile counts in place, chunk by chunk with a running carry; *count = M
__global__ void __launch_bounds__(MASK_NT) k_torso_mask_tops(int *__restrict__ tile_sums, uint32_t n_tiles, int32_t *__restrict__ count) {
    __shared__ int sw[65];
    int carry = 0;
    for (uint32_t c0 = 0; c0 < n_tiles; c0 += MASK_TILE) {
        const uint32_t base = c0 + threadIdx.x * MASK_ITEMS;
        int v[MASK_ITEMS], s = 0;
#pragma unroll
        for (int i = 0; i < MASK_ITEMS; ++i) {
            v[i] = base + i < n_tiles ? tile_sums[base + i] : 0;
            s += v[i];
        }
        int total;
        int ex = block_exclusive_scan(s, sw, total) + carry;
#pragma unroll
        for (int i = 0; i < MASK_ITEMS; ++i) {
            if (base + i < n_tiles) tile_sums[base + i] = ex;
            ex += v[i];
        }
        carry += total;
    }
    if (threadIdx.x == 0) *count = carry;
}

// pass 3: tile-local scan of the flags + the tile's base -> slot, idx and the gathers
__global__ void __launch_bounds__(MASK_NT) k_torso_mask_apply(const float2 *__restrict__ xy, const float *__restrict__ image,
                                                              const float *__restrict__ wsum, uint32_t N, const int *__restrict__ tile_base,
                                                              int32_t *__restrict__ slot, int32_t *__restrict__ idx, float2 *__restrict__ xy_m,
                                                              float *__restrict__ image_m, float *__restrict__ wsum_m) {
    __shared__ int sw[65];
    const uint32_t base = blockIdx.x * MASK_TILE + threadIdx.x * MASK_ITEMS;
    int v[MASK_ITEMS], s = 0;
#pragma unroll
    for (int i = 0; i < MASK_ITEMS; ++i) {
        v[i] = base + i < N ? slot[base + i] : 0;
        s += v[i];
    }
    int total;
    int pos = block_exclusive_scan(s, sw, total) + tile_base[blockIdx.x];
#pragma unroll
    for (int i = 0; i < MASK_ITEMS; ++i) {
        const uint32_t p = base + i;
        if (p >= N) break;
        slot[p] = v[i] ? pos : -1;
        if (v[i]) {
            idx[pos] = (int32_t)p;
            xy_m[pos] = xy[p];
            if (image) {
                image_m[3 * (size_t)pos + 0] = image[3 * (size_t)p + 0];
                image_m[3 * (size_t)pos + 1] = image[3 * (size_t)p + 1];
                image_m[3 * (size_t)pos + 2] = image[3 * (size_t)p + 2];
                wsum_m[pos] = wsum[p];
            }
            ++pos;
        }
    }
}

// background channel k of pixel i: mode 0 the scalar 1 (bg_color = None), 1 one colour, 2 one colour per pixel
__device__ __forceinline__ float bg_at(const float *__restrict__ bg, uint32_t mode, uint32_t i, int k) {
    return mode == 0 ? 1.0f : mode == 1 ? bg[k] : bg[3 * (size_t)i + k];
}

// torch.clamp(x, 0, 1): NaN passes through
__device__ __forceinline__ float clamp01(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }

__global__ void k_torso_composite_fwd(const int32_t *__restrict__ slot, uint32_t N, const float *__restrict__ alpha,
                                      const float *__restrict__ color, const float *__restrict__ image, const float *__restrict__ wsum,
                                      const float *__restrict__ bg, uint32_t bg_mode, float *__restrict__ torso_alpha_map,
                                      float *__restrict__ torso_rgb_map, float *__restrict__ rgb_map) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
        const int s = slot[i];
        const float a = s >= 0 ? alpha[s] : 0.f;
        const float one_a = __fsub_rn(1.0f, a);                 // 1 - torso_alpha
        const float one_w = __fsub_rn(1.0f, wsum[i]);           // 1 - weights_sum
        torso_alpha_map[i] = a;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float c = s >= 0 ? color[3 * (size_t)s + k] : 0.f;
            const float t = __fadd_rn(__fmul_rn(c, a), __fmul_rn(bg_at(bg, bg_mode, i, k), one_a));   // c*a + bg*(1-a)
            torso_rgb_map[3 * (size_t)i + k] = t;
            rgb_map[3 * (size_t)i + k] = clamp01(__fadd_rn(image[3 * (size_t)i + k], __fmul_rn(one_w, t)));   // image + (1-ws)*t
        }
    }
}

__global__ void k_torso_composite_bwd(const int32_t *__restrict__ idx, uint32_t M, const float *__restrict__ alpha,
                                      const float *__restrict__ color, const float *__restrict__ image, const float *__restrict__ wsum,
                                      const float *__restrict__ bg, uint32_t bg_mode, const float *__restrict__ g_ta,
                                      const float *__restrict__ g_trgb, const float *__restrict__ g_rgb, float *__restrict__ grad_alpha,
                                      float *__restrict__ grad_color) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < M; j += gridDim.x * blockDim.x) {
        const uint32_t i = (uint32_t)idx[j];
        const float a = alpha[j];
        const float one_a = __fsub_rn(1.0f, a);
        const float one_w = __fsub_rn(1.0f, wsum[i]);
        float ga_c = 0.f, ga_bg = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float c = color[3 * (size_t)j + k];
            const float b = bg_at(bg, bg_mode, i, k);
            float gt = g_trgb ? g_trgb[3 * (size_t)i + k] : 0.f;
            if (g_rgb) {
                // the forward's pre-clamp value; torch.clamp passes the gradient where 0 <= x <= 1
                const float x = __fadd_rn(image[3 * (size_t)i + k], __fmul_rn(one_w, __fadd_rn(__fmul_rn(c, a), __fmul_rn(b, one_a))));
                if (x >= 0.f && x <= 1.f) gt = __fadd_rn(gt, __fmul_rn(g_rgb[3 * (size_t)i + k], one_w));
            }
            grad_color[3 * (size_t)j + k] = __fmul_rn(gt, a);
            ga_c = __fadd_rn(ga_c, __fmul_rn(gt, c));
            ga_bg = __fadd_rn(ga_bg, __fmul_rn(gt, b));
        }
        const float g0 = g_ta ? g_ta[i] : 0.f;
        grad_alpha[j] = __fsub_rn(__fadd_rn(g0, ga_c), ga_bg);   // d/da of c*a + bg*(1-a), plus the map's own gradient
    }
}

}  // namespace

uint32_t torso_mask_tiles(uint32_t N) { return (N + MASK_TILE - 1) / MASK_TILE; }

cudaError_t launch_torso_mask(const float *grid, uint32_t G, float thr, const float *xy, const float *image, const float *wsum, uint32_t N,
                              int32_t *idx, int32_t *slot, float *xy_m, float *image_m, float *wsum_m, int32_t *count, int *tile_sums,
                              cudaStream_t st) {
    const uint32_t n_tiles = torso_mask_tiles(N);
    k_torso_mask_count<<<n_tiles, MASK_NT, 0, st>>>(grid, (int)G, thr, (const float2 *)xy, N, slot, tile_sums);
    k_torso_mask_tops<<<1, MASK_NT, 0, st>>>(tile_sums, n_tiles, count);
    k_torso_mask_apply<<<n_tiles, MASK_NT, 0, st>>>((const float2 *)xy, image, wsum, N, tile_sums, slot, idx, (float2 *)xy_m, image_m, wsum_m);
    return cudaGetLastError();
}

cudaError_t launch_torso_composite_fwd(const int32_t *slot, uint32_t N, const float *alpha, const float *color, const float *image,
                                       const float *wsum, const float *bg, uint32_t bg_mode, float *torso_alpha_map, float *torso_rgb_map,
                                       float *rgb_map, cudaStream_t st) {
    k_torso_composite_fwd<<<grid_for(N, 256), 256, 0, st>>>(slot, N, alpha, color, image, wsum, bg, bg_mode, torso_alpha_map, torso_rgb_map,
                                                            rgb_map);
    return cudaGetLastError();
}

cudaError_t launch_torso_composite_bwd(const int32_t *idx, uint32_t M, const float *alpha, const float *color, const float *image,
                                       const float *wsum, const float *bg, uint32_t bg_mode, const float *g_ta, const float *g_trgb,
                                       const float *g_rgb, float *grad_alpha, float *grad_color, cudaStream_t st) {
    k_torso_composite_bwd<<<grid_for(M, 256), 256, 0, st>>>(idx, M, alpha, color, image, wsum, bg, bg_mode, g_ta, g_trgb, g_rgb, grad_alpha,
                                                            grad_color);
    return cudaGetLastError();
}

}  // namespace gfpp
