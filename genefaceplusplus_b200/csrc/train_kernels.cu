// train_kernels.cu -- training-side native ops of modules/radnerfs (SURVEY.md 8(f) rank 4), sm_90a.
//
// Replaces, entry point for entry point (include/gfpp.h section D):
//   march_rays_train / _backward              raymarching.cu:352-598
//   composite_rays_train_forward / _backward  raymarching.cu:603-822
//   grid_encode_forward with dy_dx, grid_encode_backward, grad_total_variation   gridencoder.cu:87-368, 505-609
//   packbits / morton3D / morton3D_invert / morton3D_dilation / sph_from_ray      raymarching.cu:162-342 (update_extra_state)
//
// What is done differently from the reference's one-thread-per-element kernels:
//   * march_rays_train is DETERMINISTIC: pass 1 counts the samples of every ray, a device-wide exclusive scan hands out the
//     point offsets in ray order, pass 2 writes.  The reference hands offsets out with atomicAdd in arrival order
//     (raymarching.cu:445-446), so its sample layout changes from run to run; ours is one of the layouts it can produce,
//     always the same one (reproducible training steps, bit-comparable with the CPU checker).
//   * compositing is one WARP per ray: lanes take consecutive samples (coalesced 128-byte loads along the ray), the
//     transmittance is a multiplicative warp-shuffle scan, the colour / weight prefix sums additive shuffle scans, the
//     T_thresh cut a ballot.  Forward and backward share the scan.
//   * the table gradient is scattered with vector reductions (one red.global.add.v2.f32 per corner for the C = 2 tables),
//     level-major so that a warp's atomics fall into one level's table.
// Marching reuses the bit-exact device marcher of the inference path (common.cuh).
#include "common.cuh"
#include "launch.cuh"
#include "ops.cuh"

namespace gfpp {

namespace {

constexpr int SCAN_NT = 1024, SCAN_ITEMS = 4, SCAN_TILE = SCAN_NT * SCAN_ITEMS;

__device__ __forceinline__ float ray_t0(const MarchConst &mc, float near, float noise) {
    // t0 = near + clamp(near * dt_gamma, dt_min, dt_max) * noise   (raymarching.cu:391-392)
    return __fadd_rn(near, __fmul_rn(step_len(mc, near), noise));
}

// ---- pass 1: samples per ray ----
__global__ void k_march_train_count(MarchConst mc, const float *__restrict__ rays_o, const float *__restrict__ rays_d,
                                    const float *__restrict__ nears, const float *__restrict__ fars, const float *__restrict__ noises,
                                    uint32_t N, uint32_t max_steps, int *__restrict__ rays) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        RayGeom g;
        ray_geom_init(g, rays_o[3 * n], rays_o[3 * n + 1], rays_o[3 * n + 2], rays_d[3 * n], rays_d[3 * n + 1], rays_d[3 * n + 2]);
        const float far = fars[n];
        float t = ray_t0(mc, nears[n], noises[n]);
        uint32_t steps = 0;
        float x, y, z, dt;
        while (steps < max_steps && march_next(mc, g, far, t, x, y, z, dt)) ++steps;
        rays[3 * n] = (int)n;
        rays[3 * n + 2] = (int)steps;
    }
}

// ---- exclusive scan of rays[.,2] into rays[.,1]: tile sums, scan of the tile sums (one CTA), tile-local scan + base ----
__global__ void __launch_bounds__(SCAN_NT) k_scan_tile_sums(const int *__restrict__ rays, uint32_t N, int *__restrict__ tile_sums) {
    __shared__ int sw[65];
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    int v = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i)
        if (base + i < N) v += rays[3 * (size_t)(base + i) + 2];
    int total;
    (void)block_exclusive_scan(v, sw, total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// one CTA: exclusive scan of up to SCAN_TILE tile sums (N <= SCAN_TILE^2 = 16.7 M rays); also bumps the reference's counter
__global__ void __launch_bounds__(SCAN_NT) k_scan_tops(int *__restrict__ tile_sums, uint32_t n_tiles, uint32_t N, int *__restrict__ counter) {
    __shared__ int sw[65];
    const uint32_t base = threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = base + i < n_tiles ? tile_sums[base + i] : 0;
        s += v[i];
    }
    int total;
    int ex = block_exclusive_scan(s, sw, total);
    const int start = counter[0];   // the reference keeps accumulating into `counter` (atomicAdd): offsets start there
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        if (base + i < n_tiles) tile_sums[base + i] = start + ex;
        ex += v[i];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        counter[0] = start + total;
        counter[1] += (int)N;
    }
}

__global__ void __launch_bounds__(SCAN_NT) k_scan_apply(int *__restrict__ rays, uint32_t N, const int *__restrict__ tile_base) {
    __shared__ int sw[65];
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = base + i < N ? rays[3 * (size_t)(base + i) + 2] : 0;
        s += v[i];
    }
    int total;
    int ex = block_exclusive_scan(s, sw, total) + tile_base[blockIdx.x];
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        if (base + i < N) rays[3 * (size_t)(base + i) + 1] = ex;
        ex += v[i];
    }
}

// ---- pass 2: write the samples of every ray at its offset ----
__global__ void k_march_train_write(MarchConst mc, const float *__restrict__ rays_o, const float *__restrict__ rays_d,
                                    const float *__restrict__ nears, const float *__restrict__ fars, const float *__restrict__ noises,
                                    uint32_t N, uint32_t M, const int *__restrict__ rays, float *__restrict__ xyzs,
                                    float *__restrict__ dirs, float *__restrict__ deltas) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        const uint32_t off = (uint32_t)rays[3 * n + 1], ns = (uint32_t)rays[3 * n + 2];
        if (ns == 0 || off + ns > M) continue;   // raymarching.cu:455-456
        RayGeom g;
        ray_geom_init(g, rays_o[3 * n], rays_o[3 * n + 1], rays_o[3 * n + 2], rays_d[3 * n], rays_d[3 * n + 1], rays_d[3 * n + 2]);
        const float far = fars[n];
        float t = ray_t0(mc, nears[n], noises[n]);
        float x, y, z, dt;
        for (uint32_t s = 0; s < ns && march_next(mc, g, far, t, x, y, z, dt); ++s) {
            const size_t p = (size_t)off + s;
            xyzs[3 * p] = x; xyzs[3 * p + 1] = y; xyzs[3 * p + 2] = z;
            dirs[3 * p] = g.dx; dirs[3 * p + 1] = g.dy; dirs[3 * p + 2] = g.dz;
            deltas[2 * p] = dt; deltas[2 * p + 1] = t;   // t already advanced past the sample (:497-499)
        }
    }
}

// ---- march_rays_train_backward: xyz = o + t d  =>  d/do = 1, d/dd = t (+ the direct dirs gradient); one warp per ray ----
__global__ void k_march_train_backward(const float *__restrict__ grad_xyzs, const float *__restrict__ grad_dirs, const int *__restrict__ rays,
                                       const float *__restrict__ deltas, uint32_t N, uint32_t M, float *__restrict__ grad_rays_o,
                                       float *__restrict__ grad_rays_d) {
    const int lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; n < N; n += warps) {
        const uint32_t off = (uint32_t)rays[3 * n + 1], ns = (uint32_t)rays[3 * n + 2];
        if (ns == 0 || off + ns > M) continue;
        float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
        for (uint32_t s = lane; s < ns; s += 32) {
            const size_t p = (size_t)off + s;
            const float t = deltas[2 * p + 1];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float gx = grad_xyzs[3 * p + c];
                go[c] += gx;
                gd[c] += gx * t + grad_dirs[3 * p + c];
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                go[c] += __shfl_xor_sync(0xffffffffu, go[c], o);
                gd[c] += __shfl_xor_sync(0xffffffffu, gd[c], o);
            }
        }
        if (lane < 3) {   // the reference accumulates into row n of grad_rays_* (thread id, not rays[n].index: :548-549)
            grad_rays_o[3 * (size_t)n + lane] += lane == 0 ? go[0] : lane == 1 ? go[1] : go[2];
            grad_rays_d[3 * (size_t)n + lane] += lane == 0 ? gd[0] : lane == 1 ? gd[1] : gd[2];
        }
    }
}

// ---- warp-level scans along a ray ----
__device__ __forceinline__ float warp_inclusive_prod(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v *= u;
    }
    return v;
}
__device__ __forceinline__ float warp_inclusive_sum(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    return v;
}

// One warp per ray, 32 samples per trip.  BACKWARD == false: kernel_composite_rays_train_forward (raymarching.cu:603-688);
// true: kernel_composite_rays_train_backward (:711-810).  Sample k of a ray is processed iff every earlier sample left
// T >= T_thresh (the reference breaks AFTER accumulating the sample that drops T below the threshold).
template <bool BACKWARD>
__global__ void k_composite_train(const float *__restrict__ sigmas, const float *__restrict__ rgbs, const float *__restrict__ ambient,
                                  const float *__restrict__ deltas, const int *__restrict__ rays, uint32_t M, uint32_t N, float T_thresh,
                                  float *__restrict__ weights_sum, float *__restrict__ ambient_sum, float *__restrict__ depth,
                                  float *__restrict__ image, const float *__restrict__ grad_weights_sum,
                                  const float *__restrict__ grad_ambient_sum, const float *__restrict__ grad_image,
                                  float *__restrict__ grad_sigmas, float *__restrict__ grad_rgbs, float *__restrict__ grad_ambient) {
    const int lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; n < N; n += warps) {
        const uint32_t index = (uint32_t)rays[3 * n], off = (uint32_t)rays[3 * n + 1], ns = (uint32_t)rays[3 * n + 2];
        const bool empty = ns == 0 || off + ns > M;
        if (empty) {
            if (!BACKWARD && lane == 0) {
                weights_sum[index] = 0.f; ambient_sum[index] = 0.f; depth[index] = 0.f;
                image[3 * (size_t)index] = 0.f; image[3 * (size_t)index + 1] = 0.f; image[3 * (size_t)index + 2] = 0.f;
            }
            continue;
        }
        float gi0 = 0.f, gi1 = 0.f, gi2 = 0.f, gws = 0.f, gamb = 0.f, rf = 0.f, gf = 0.f, bf = 0.f, wsf = 0.f;
        if (BACKWARD) {
            gi0 = grad_image[3 * (size_t)index]; gi1 = grad_image[3 * (size_t)index + 1]; gi2 = grad_image[3 * (size_t)index + 2];
            gws = grad_weights_sum[index]; gamb = grad_ambient_sum[index];
            rf = image[3 * (size_t)index]; gf = image[3 * (size_t)index + 1]; bf = image[3 * (size_t)index + 2];
            wsf = weights_sum[index];
        }
        float T_in = 1.0f, r_in = 0.f, g_in = 0.f, b_in = 0.f, ws_in = 0.f, d_in = 0.f, amb_in = 0.f;
        for (uint32_t s0 = 0; s0 < ns; s0 += 32) {
            const uint32_t s = s0 + lane;
            const bool have = s < ns;
            const size_t p = (size_t)off + (have ? s : 0);
            const float sg = have ? sigmas[p] : 0.f, dt = have ? deltas[2 * p] : 0.f, tt = have ? deltas[2 * p + 1] : 0.f;
            const float c0 = have ? rgbs[3 * p] : 0.f, c1 = have ? rgbs[3 * p + 1] : 0.f, c2 = have ? rgbs[3 * p + 2] : 0.f;
            const float alpha = have ? 1.0f - __expf(-sg * dt) : 0.f;
            const float P = warp_inclusive_prod(1.0f - alpha, lane);          // prod_{j<=lane} (1 - alpha_j)
            float P_prev = __shfl_up_sync(0xffffffffu, P, 1);
            if (lane == 0) P_prev = 1.0f;
            const float T_before = T_in * P_prev, T_after = T_in * P;
            // first sample of this trip that drops T below the threshold: it is the last one processed
            const unsigned cut = __ballot_sync(0xffffffffu, have && T_after < T_thresh);
            const int last = cut ? __ffs(cut) - 1 : 31;
            const bool live = have && lane <= last;
            const float w = live ? alpha * T_before : 0.f;
            const float r = r_in + warp_inclusive_sum(w * c0, lane), g = g_in + warp_inclusive_sum(w * c1, lane),
                        b = b_in + warp_inclusive_sum(w * c2, lane), ws = ws_in + warp_inclusive_sum(w, lane);
            if (BACKWARD) {
                if (live) {
                    grad_rgbs[3 * p] = gi0 * w; grad_rgbs[3 * p + 1] = gi1 * w; grad_rgbs[3 * p + 2] = gi2 * w;
                    grad_ambient[p] = gamb;
                    grad_sigmas[p] = dt * (gi0 * (T_after * c0 - (rf - r)) + gi1 * (T_after * c1 - (gf - g)) + gi2 * (T_after * c2 - (bf - b)) +
                                           gws * (1.0f - wsf));
                }
            } else {
                d_in += warp_inclusive_sum(w * tt, lane);                      // valid in lane 31 only; broadcast below
                amb_in += warp_inclusive_sum(live ? ambient[p] : 0.f, lane);
                d_in = __shfl_sync(0xffffffffu, d_in, 31);
                amb_in = __shfl_sync(0xffffffffu, amb_in, 31);
            }
            r_in = __shfl_sync(0xffffffffu, r, 31); g_in = __shfl_sync(0xffffffffu, g, 31); b_in = __shfl_sync(0xffffffffu, b, 31);
            ws_in = __shfl_sync(0xffffffffu, ws, 31);
            T_in = __shfl_sync(0xffffffffu, T_after, last);
            if (cut) break;
        }
        if (!BACKWARD && lane == 0) {
            weights_sum[index] = ws_in; ambient_sum[index] = amb_in; depth[index] = d_in;
            image[3 * (size_t)index] = r_in; image[3 * (size_t)index + 1] = g_in; image[3 * (size_t)index + 2] = b_in;
        }
    }
}

// ---- grid encoder, training side (D in {2,3}, C = 2) ----
__device__ __forceinline__ float smoothstep_d(float x) { return 6.0f * x * (1.0f - x); }

template <int D>
__device__ __forceinline__ bool cell_of_input(const GridMeta &gm, int l, const float *in, uint32_t (&pg)[3], float (&pos)[3], float (&deriv)[3]) {
#pragma unroll
    for (int d = 0; d < D; ++d)
        if (in[d] < 0.f || in[d] > 1.f) return false;
    const float s = gm.scale[l];
    pg[2] = 0u; pos[2] = 0.f; deriv[2] = 1.f;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        float p = __fadd_rn(__fmul_rn(in[d], s), gm.align_off);
        const float f0 = floorf(p);
        pg[d] = (uint32_t)f0;
        p -= f0;
        deriv[d] = 1.0f;
        if (gm.interp == 1) { deriv[d] = smoothstep_d(p); p = p * p * (3.0f - 2.0f * p); }
        pos[d] = p;
    }
    return true;
}

// forward with dy_dx [B, L, D, 2] (gridencoder.cu:87-243): outputs through the same lookups as the inference op
template <int D>
__global__ void k_grid_encode_dydx(GridMeta gm, const float *__restrict__ inputs, const float2 *__restrict__ table,
                                   float2 *__restrict__ outputs, float2 *__restrict__ dy_dx, uint32_t B) {
    const uint32_t L = gm.num_levels, total = B * L;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t l = i / B, b = i - l * B;
        float in[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int d = 0; d < D; ++d) in[d] = inputs[(size_t)b * D + d];
        outputs[(size_t)l * B + b] = D == 3 ? grid_lookup3(gm, table, l, in[0], in[1], in[2]) : grid_lookup2(gm, table, l, in[0], in[1]);
        float2 *dd = dy_dx + ((size_t)b * L + l) * D;
        uint32_t pg[3];
        float pos[3], deriv[3];
        if (!cell_of_input<D>(gm, l, in, pg, pos, deriv)) {
#pragma unroll
            for (int d = 0; d < D; ++d) dd[d] = make_float2(0.f, 0.f);
            continue;
        }
        const float2 *tb = table + gm.offset[l];
        const float s = gm.scale[l];
#pragma unroll
        for (int gd = 0; gd < D; ++gd) {
            float2 acc = make_float2(0.f, 0.f);
#pragma unroll
            for (int idx = 0; idx < (1 << (D - 1)); ++idx) {
                float w = s;
                uint32_t pl[3] = {pg[0], pg[1], pg[2]};
#pragma unroll
                for (int nd = 0; nd < D - 1; ++nd) {
                    const int d = nd >= gd ? nd + 1 : nd;
                    if ((idx & (1 << nd)) == 0) w *= 1.0f - pos[d];
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                pl[gd] = pg[gd];
                const float2 lft = __ldg(tb + grid_slot(gm, l, pl[0], pl[1], pl[2]));
                pl[gd] = pg[gd] + 1;
                const float2 rgt = __ldg(tb + grid_slot(gm, l, pl[0], pl[1], pl[2]));
                acc.x += w * (rgt.x - lft.x) * deriv[gd];
                acc.y += w * (rgt.y - lft.y) * deriv[gd];
            }
            dd[gd] = acc;
        }
    }
}

// table gradient: grad [L,B,2] scattered to the 2^D corners with one vector reduction each (gridencoder.cu:246-340)
template <int D>
__global__ void k_grid_backward(GridMeta gm, const float2 *__restrict__ grad, const float *__restrict__ inputs, float2 *__restrict__ grad_table,
                                uint32_t B) {
    const uint32_t total = B * gm.num_levels;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t l = i / B, b = i - l * B;
        float in[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int d = 0; d < D; ++d) in[d] = inputs[(size_t)b * D + d];
        uint32_t pg[3];
        float pos[3], deriv[3];
        if (!cell_of_input<D>(gm, l, in, pg, pos, deriv)) continue;   // grad is zero-initialised by the caller
        const float2 g = grad[(size_t)l * B + b];
        float2 *gt = grad_table + gm.offset[l];
#pragma unroll
        for (int idx = 0; idx < (1 << D); ++idx) {
            float w = 1.0f;
            uint32_t pl[3] = {pg[0], pg[1], pg[2]};
#pragma unroll
            for (int d = 0; d < D; ++d) {
                if ((idx & (1 << d)) == 0) w *= 1.0f - pos[d];
                else { w *= pos[d]; pl[d] = pg[d] + 1; }
            }
            atomicAdd(gt + grid_slot(gm, l, pl[0], pl[1], pl[2]), make_float2(w * g.x, w * g.y));   // red.global.add.v2.f32
        }
    }
}

// input gradient from dy_dx (gridencoder.cu:343-368)
__global__ void k_grid_input_backward(const float2 *__restrict__ grad, const float2 *__restrict__ dy_dx, float *__restrict__ grad_inputs,
                                      uint32_t B, uint32_t D, uint32_t L) {
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < B * D; t += gridDim.x * blockDim.x) {
        const uint32_t b = t / D, d = t - b * D;
        const float2 *dd = dy_dx + (size_t)b * L * D;
        float r = 0.f;
        for (uint32_t l = 0; l < L; ++l) {
            const float2 g = grad[(size_t)l * B + b], y = dd[(size_t)l * D + d];
            r += g.x * y.x;
            r += g.y * y.y;
        }
        grad_inputs[t] = r;
    }
}

// total-variation gradient of the cells the inputs fall into (gridencoder.cu:505-592)
template <int D>
__global__ void k_grad_tv(GridMeta gm, const float *__restrict__ inputs, const float2 *__restrict__ table, float2 *__restrict__ grad_table,
                          float weight, uint32_t B) {
    const uint32_t total = B * gm.num_levels;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t l = i / B, b = i - l * B;
        float in[3] = {0.f, 0.f, 0.f};
        bool oob = false;
#pragma unroll
        for (int d = 0; d < D; ++d) {
            in[d] = inputs[(size_t)b * D + d];
            if (in[d] < 0.f || in[d] > 1.f) oob = true;
        }
        if (oob) continue;
        const float s = gm.scale[l];
        const uint32_t res = (uint32_t)ceilf(s) + 1u;
        uint32_t pg[3] = {0u, 0u, 0u};
#pragma unroll
        for (int d = 0; d < D; ++d) pg[d] = (uint32_t)floorf(__fadd_rn(__fmul_rn(in[d], s), gm.align_off));
        const float2 *tb = table + gm.offset[l];
        const uint32_t index = grid_slot(gm, l, pg[0], pg[1], pg[2]);
        const float2 c = __ldg(tb + index);
        float2 sum = make_float2(0.f, 0.f), sq = make_float2(0.f, 0.f);
#pragma unroll
        for (int d = 0; d < D; ++d) {
            const uint32_t cur = pg[d];
            if (cur < res) {
                pg[d] = cur + 1;
                const float2 o = __ldg(tb + grid_slot(gm, l, pg[0], pg[1], pg[2]));
                const float gx = c.x - o.x, gy = c.y - o.y;
                sum.x += gx; sum.y += gy; sq.x += gx * gx; sq.y += gy * gy;
            }
            if (cur > 0) {
                pg[d] = cur - 1;
                const float2 o = __ldg(tb + grid_slot(gm, l, pg[0], pg[1], pg[2]));
                const float gx = c.x - o.x, gy = c.y - o.y;
                sum.x += gx; sum.y += gy; sq.x += gx * gx; sq.y += gy * gy;
            }
            pg[d] = cur;
        }
        const float w = weight / (float)(2 * D);
        atomicAdd(grad_table + gm.offset[l] + index, make_float2(w * sum.x * rsqrtf(sq.x + 1e-9f), w * sum.y * rsqrtf(sq.y + 1e-9f)));
    }
}

// ---- update_extra_state helpers ----

__global__ void k_packbits(const float *__restrict__ grid, uint32_t N, float thresh, uint8_t *__restrict__ bitfield) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        const float4 a = *reinterpret_cast<const float4 *>(grid + (size_t)n * 8), b = *reinterpret_cast<const float4 *>(grid + (size_t)n * 8 + 4);
        uint32_t bits = 0;
        bits |= a.x > thresh ? 1u : 0u; bits |= a.y > thresh ? 2u : 0u; bits |= a.z > thresh ? 4u : 0u; bits |= a.w > thresh ? 8u : 0u;
        bits |= b.x > thresh ? 16u : 0u; bits |= b.y > thresh ? 32u : 0u; bits |= b.z > thresh ? 64u : 0u; bits |= b.w > thresh ? 128u : 0u;
        bitfield[n] = (uint8_t)bits;
    }
}

__global__ void k_morton3D(const int *__restrict__ coords, uint32_t N, int *__restrict__ indices) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x)
        indices[n] = (int)morton3((uint32_t)coords[3 * n], (uint32_t)coords[3 * n + 1], (uint32_t)coords[3 * n + 2]);
}

__global__ void k_morton3D_invert(const int *__restrict__ indices, uint32_t N, int *__restrict__ coords) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        const uint32_t ind = (uint32_t)indices[n];
        coords[3 * n] = (int)compact3(ind); coords[3 * n + 1] = (int)compact3(ind >> 1); coords[3 * n + 2] = (int)compact3(ind >> 2);
    }
}

__global__ void k_morton3D_dilation(const float *__restrict__ grid, uint32_t C, uint32_t H, float *__restrict__ out) {
    const uint32_t H3 = H * H * H, total = C * H3;
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < total; n += gridDim.x * blockDim.x) {
        const uint32_t c = n / H3, ind = n - c * H3;
        const uint32_t x = compact3(ind), y = compact3(ind >> 1), z = compact3(ind >> 2);
        const float *g = grid + (size_t)c * H3;
        float r = grid[n];
        if (x + 1 < H) r = fmaxf(r, g[morton3(x + 1, y, z)]);
        if (x > 0) r = fmaxf(r, g[morton3(x - 1, y, z)]);
        if (y + 1 < H) r = fmaxf(r, g[morton3(x, y + 1, z)]);
        if (y > 0) r = fmaxf(r, g[morton3(x, y - 1, z)]);
        if (z + 1 < H) r = fmaxf(r, g[morton3(x, y, z + 1)]);
        if (z > 0) r = fmaxf(r, g[morton3(x, y, z - 1)]);
        out[n] = r;
    }
}

__global__ void k_sph_from_ray(const float *__restrict__ rays_o, const float *__restrict__ rays_d, float radius, uint32_t N,
                               float *__restrict__ coords) {
    const float rpi = 0.3183098861837907f;
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
        const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
        const float A = dx * dx + dy * dy + dz * dz;
        const float Bq = ox * dx + oy * dy + oz * dz;   // B / 2
        const float Cq = ox * ox + oy * oy + oz * oz - radius * radius;
        const float t = (-Bq + sqrtf(Bq * Bq - A * Cq)) / A;   // the larger (positive) root
        const float x = ox + t * dx, y = oy + t * dy, z = oz + t * dz;
        coords[2 * n] = 2.0f * atan2f(sqrtf(x * x + z * z), y) * rpi - 1.0f;
        coords[2 * n + 1] = atan2f(z, x) * rpi;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ launchers
size_t march_train_scratch_bytes(uint32_t N) { return ((size_t)(N + SCAN_TILE - 1) / SCAN_TILE + 1) * sizeof(int); }

cudaError_t launch_march_rays_train(const MarchConst &mc, const float *rays_o, const float *rays_d, const float *nears, const float *fars,
                                    const float *noises, uint32_t N, uint32_t M, uint32_t max_steps, float *xyzs, float *dirs, float *deltas,
                                    int *rays, int *counter, int *scratch, int *n_launches, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    const uint32_t n_tiles = (N + SCAN_TILE - 1) / SCAN_TILE;
    if (n_tiles > (uint32_t)SCAN_TILE) return cudaErrorInvalidValue;
    k_march_train_count<<<grid_for(N, 128), 128, 0, st>>>(mc, rays_o, rays_d, nears, fars, noises, N, max_steps, rays);
    k_scan_tile_sums<<<n_tiles, SCAN_NT, 0, st>>>(rays, N, scratch);
    k_scan_tops<<<1, SCAN_NT, 0, st>>>(scratch, n_tiles, N, counter);
    k_scan_apply<<<n_tiles, SCAN_NT, 0, st>>>(rays, N, scratch);
    k_march_train_write<<<grid_for(N, 128), 128, 0, st>>>(mc, rays_o, rays_d, nears, fars, noises, N, M, rays, xyzs, dirs, deltas);
    if (n_launches) *n_launches = 5;
    return cudaGetLastError();
}

cudaError_t launch_march_rays_train_backward(const float *grad_xyzs, const float *grad_dirs, const int *rays, const float *deltas, uint32_t N,
                                             uint32_t M, float *grad_rays_o, float *grad_rays_d, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_march_train_backward<<<grid_for((uint64_t)N * 32, 256), 256, 0, st>>>(grad_xyzs, grad_dirs, rays, deltas, N, M, grad_rays_o, grad_rays_d);
    return cudaGetLastError();
}

cudaError_t launch_composite_train_forward(const float *sigmas, const float *rgbs, const float *ambient, const float *deltas, const int *rays,
                                           uint32_t M, uint32_t N, float T_thresh, float *weights_sum, float *ambient_sum, float *depth,
                                           float *image, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_composite_train<false><<<grid_for((uint64_t)N * 32, 256), 256, 0, st>>>(sigmas, rgbs, ambient, deltas, rays, M, N, T_thresh, weights_sum,
                                                                              ambient_sum, depth, image, nullptr, nullptr, nullptr, nullptr,
                                                                              nullptr, nullptr);
    return cudaGetLastError();
}

cudaError_t launch_composite_train_backward(const float *grad_weights_sum, const float *grad_ambient_sum, const float *grad_image,
                                            const float *sigmas, const float *rgbs, const float *ambient, const float *deltas, const int *rays,
                                            const float *weights_sum, const float *ambient_sum, const float *image, uint32_t M, uint32_t N,
                                            float T_thresh, float *grad_sigmas, float *grad_rgbs, float *grad_ambient, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_composite_train<true><<<grid_for((uint64_t)N * 32, 256), 256, 0, st>>>(
        sigmas, rgbs, ambient, deltas, rays, M, N, T_thresh, const_cast<float *>(weights_sum), const_cast<float *>(ambient_sum), nullptr,
        const_cast<float *>(image), grad_weights_sum, grad_ambient_sum, grad_image, grad_sigmas, grad_rgbs, grad_ambient);
    return cudaGetLastError();
}

cudaError_t launch_grid_encode_dydx(const GridMeta &gm, const float *inputs, const float *table, float *outputs, float *dy_dx, uint32_t B,
                                    cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    const uint32_t total = B * gm.num_levels;
    if (gm.dim == 3)
        k_grid_encode_dydx<3><<<grid_for(total, 256), 256, 0, st>>>(gm, inputs, (const float2 *)table, (float2 *)outputs, (float2 *)dy_dx, B);
    else
        k_grid_encode_dydx<2><<<grid_for(total, 256), 256, 0, st>>>(gm, inputs, (const float2 *)table, (float2 *)outputs, (float2 *)dy_dx, B);
    return cudaGetLastError();
}

cudaError_t launch_grid_backward(const GridMeta &gm, const float *grad, const float *inputs, float *grad_table, const float *dy_dx,
                                 float *grad_inputs, uint32_t B, int *n_launches, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    const uint32_t total = B * gm.num_levels;
    if (gm.dim == 3) k_grid_backward<3><<<grid_for(total, 256), 256, 0, st>>>(gm, (const float2 *)grad, inputs, (float2 *)grad_table, B);
    else k_grid_backward<2><<<grid_for(total, 256), 256, 0, st>>>(gm, (const float2 *)grad, inputs, (float2 *)grad_table, B);
    int n = 1;
    if (dy_dx && grad_inputs) {
        k_grid_input_backward<<<grid_for((uint64_t)B * gm.dim, 256), 256, 0, st>>>((const float2 *)grad, (const float2 *)dy_dx, grad_inputs, B,
                                                                                  gm.dim, gm.num_levels);
        n = 2;
    }
    if (n_launches) *n_launches = n;
    return cudaGetLastError();
}

cudaError_t launch_grad_tv(const GridMeta &gm, const float *inputs, const float *table, float *grad_table, float weight, uint32_t B,
                           cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    const uint32_t total = B * gm.num_levels;
    if (gm.dim == 3) k_grad_tv<3><<<grid_for(total, 256), 256, 0, st>>>(gm, inputs, (const float2 *)table, (float2 *)grad_table, weight, B);
    else k_grad_tv<2><<<grid_for(total, 256), 256, 0, st>>>(gm, inputs, (const float2 *)table, (float2 *)grad_table, weight, B);
    return cudaGetLastError();
}

cudaError_t launch_packbits(const float *grid, uint32_t N, float thresh, uint8_t *bitfield, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_packbits<<<grid_for(N, 256), 256, 0, st>>>(grid, N, thresh, bitfield);
    return cudaGetLastError();
}
cudaError_t launch_morton3D(const int *coords, uint32_t N, int *indices, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_morton3D<<<grid_for(N, 256), 256, 0, st>>>(coords, N, indices);
    return cudaGetLastError();
}
cudaError_t launch_morton3D_invert(const int *indices, uint32_t N, int *coords, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_morton3D_invert<<<grid_for(N, 256), 256, 0, st>>>(indices, N, coords);
    return cudaGetLastError();
}
cudaError_t launch_morton3D_dilation(const float *grid, uint32_t C, uint32_t H, float *out, cudaStream_t st) {
    k_morton3D_dilation<<<grid_for((uint64_t)C * H * H * H, 256), 256, 0, st>>>(grid, C, H, out);
    return cudaGetLastError();
}
cudaError_t launch_sph_from_ray(const float *rays_o, const float *rays_d, float radius, uint32_t N, float *coords, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_sph_from_ray<<<grid_for(N, 256), 256, 0, st>>>(rays_o, rays_d, radius, N, coords);
    return cudaGetLastError();
}

}  // namespace gfpp
