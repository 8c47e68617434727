// ops_kernels.cu -- per-op kernels behind the (A) level of include/gfpp.h.
//
// These mirror the six inference ops of the reference's extensions one-to-one so that (i) the reference's
// unmodified Python wrappers can run on this library and (ii) each op can be parity-tested in isolation
// against the C oracle and against the reference's own kernels (oracle/_ref).  The production path is the
// fused renderer in head_kernel.cu / torso_kernel.cu; these kernels are simple grid-stride SIMT kernels
// sized in multiples of the SM count.
#include "common.cuh"
#include "launch.cuh"
#include "ops.cuh"

namespace gfpp {

// ---- near_far_from_aabb (raymarching.cu:91-145) ----
__global__ void k_near_far(const float *__restrict__ rays_o, const float *__restrict__ rays_d,
                           const float *__restrict__ aabb, uint32_t N, float min_near, float *__restrict__ nears,
                           float *__restrict__ fars) {
    float bb[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) bb[i] = __ldg(aabb + i);
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        RayGeom g;
        ray_geom_init(g, rays_o[3 * n], rays_o[3 * n + 1], rays_o[3 * n + 2], rays_d[3 * n], rays_d[3 * n + 1],
                      rays_d[3 * n + 2]);
        float nr, fr;
        near_far(g, bb, min_near, nr, fr);
        nears[n] = nr;
        fars[n] = fr;
    }
}

// ---- march_rays (raymarching.cu:827-929): one round, up to n_step samples per alive ray ----
__global__ void k_march_rays(MarchConst mc, uint32_t n_alive, uint32_t n_step, const int32_t *__restrict__ rays_alive,
                             const float *__restrict__ rays_t, const float *__restrict__ rays_o,
                             const float *__restrict__ rays_d, const float *__restrict__ fars, float *__restrict__ xyzs,
                             float *__restrict__ dirs, float *__restrict__ deltas, const float *__restrict__ noises) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < n_alive; n += gridDim.x * blockDim.x) {
        const int ray = rays_alive[n];
        RayGeom g;
        ray_geom_init(g, rays_o[3 * ray], rays_o[3 * ray + 1], rays_o[3 * ray + 2], rays_d[3 * ray],
                      rays_d[3 * ray + 1], rays_d[3 * ray + 2]);
        float t = rays_t[ray];
        const float far = fars[ray];
        // optional jitter (zero on the inference path): t += clamp(t*dt_gamma) * noise
        t = __fadd_rn(t, __fmul_rn(step_len(mc, t), noises[n]));
        float *px = xyzs + (size_t)n * n_step * 3, *pd = dirs + (size_t)n * n_step * 3,
              *pl = deltas + (size_t)n * n_step * 2;
        for (uint32_t s = 0; s < n_step; ++s) {
            float x, y, z, dt;
            if (!march_next(mc, g, far, t, x, y, z, dt)) break;
            px[0] = x; px[1] = y; px[2] = z;
            pd[0] = g.dx; pd[1] = g.dy; pd[2] = g.dz;
            pl[0] = dt; pl[1] = t;
            px += 3; pd += 3; pl += 2;
        }
    }
}

// ---- composite_rays (raymarching.cu:942-1029) ----
__global__ void k_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t *__restrict__ rays_alive,
                                 float *__restrict__ rays_t, const float *__restrict__ sigmas,
                                 const float *__restrict__ rgbs, const float *__restrict__ deltas,
                                 float *__restrict__ weights_sum, float *__restrict__ depth, float *__restrict__ image) {
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < n_alive; n += gridDim.x * blockDim.x) {
        const int ray = rays_alive[n];
        const float *sg = sigmas + (size_t)n * n_step, *cl = rgbs + (size_t)n * n_step * 3,
                    *dl = deltas + (size_t)n * n_step * 2;
        float t = rays_t[ray], ws = weights_sum[ray], dp = depth[ray];
        float r = image[3 * ray], g = image[3 * ray + 1], b = image[3 * ray + 2];
        uint32_t step = 0;
        while (step < n_step) {
            if (dl[0] == 0) break;
            const float alpha = 1.0f - expf(-sg[0] * dl[0]);  // accurate expf (SURVEY H6), not __expf
            const float T = 1.0f - ws;
            const float w = alpha * T;
            ws += w;
            t = dl[1];
            dp += w * t;
            r += w * cl[0];
            g += w * cl[1];
            b += w * cl[2];
            if (T < T_thresh) break;
            ++sg; cl += 3; dl += 2; ++step;
        }
        if (step < n_step) rays_alive[n] = -1;
        else rays_t[ray] = t;
        weights_sum[ray] = ws;
        depth[ray] = dp;
        image[3 * ray] = r; image[3 * ray + 1] = g; image[3 * ray + 2] = b;
    }
}

// ---- grid_encode_forward (gridencoder.cu:87-196), outputs [L,B,2] ----
template <int D>
__global__ void k_grid_encode(GridMeta gm, const float *__restrict__ inputs, const float2 *__restrict__ table,
                              float2 *__restrict__ outputs, uint32_t B) {
    const uint32_t total = B * gm.num_levels;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t l = i / B, b = i - l * B;  // level-major: a warp works on one level of neighbouring points
        float2 f;
        if (D == 3) f = grid_lookup3(gm, table, l, inputs[3 * b], inputs[3 * b + 1], inputs[3 * b + 2]);
        else f = grid_lookup2(gm, table, l, inputs[2 * b], inputs[2 * b + 1]);
        outputs[(size_t)l * B + b] = f;
    }
}

// ---- sh_encode_forward (shencoder.cu:27-68), degree <= 4 ----
__global__ void k_sh_encode(const float *__restrict__ inputs, float *__restrict__ outputs, uint32_t B, uint32_t degree) {
    const uint32_t C2 = degree * degree;
    for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
        float o[16];
        sh4(inputs[3 * b], inputs[3 * b + 1], inputs[3 * b + 2], o);
        for (uint32_t c = 0; c < C2; ++c) outputs[(size_t)b * C2 + c] = o[c];
    }
}

// ---- freq_encode_forward (freqencoder.cu:30-58); accurate sinf instead of __sinf (SURVEY H6) ----
__global__ void k_freq_encode(const float *__restrict__ inputs, uint32_t B, uint32_t D, uint32_t C,
                              float *__restrict__ outputs) {
    const uint32_t total = B * C;
    const float half_pi = 3.141592653589793f / 2;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t b = i / C, c = i - b * C;
        float v;
        if (c < D) {
            v = inputs[b * D + c];
        } else {
            const uint32_t col = c / D - 1, d = c % D, f = col / 2;
            v = sinf(__fadd_rn(scalbnf(inputs[b * D + d], (int)f), (float)(col % 2) * half_pi));
        }
        outputs[i] = v;
    }
}

// ---- tight cell bounds of the occupied voxels (used to skip bit reads in known-empty space) ----
// bounds[0..2] = min cell, bounds[3..5] = max cell over all cascades; initialised by the caller to
// {INT_MAX.., -1..}.  Cells are decoded from the Morton bit index.

__global__ void k_occupancy_bounds(const uint8_t *__restrict__ bits, uint32_t n_bytes, uint32_t H3, int *bounds) {
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {-1, -1, -1};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += gridDim.x * blockDim.x) {
        uint32_t v = bits[i];
        while (v) {
            const int k = __ffs(v) - 1;
            v &= v - 1;
            const uint32_t m = (i * 8u + k) % H3;
            const int c[3] = {(int)compact3(m), (int)compact3(m >> 1), (int)compact3(m >> 2)};
#pragma unroll
            for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], c[a]); hi[a] = max(hi[a], c[a]); }
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        if ((threadIdx.x & 31) == 0) {
            if (lo[a] != INT_MAX) atomicMin(bounds + a, lo[a]);
            if (hi[a] >= 0) atomicMax(bounds + 3 + a, hi[a]);
        }
    }
}

// ---- coarse occupancy: bit (c*Hc^3 + (cx*Hc + cy)*Hc + cz) = OR of the 4x4x4 fine cells (Morton-indexed bitfield) ----
__global__ void k_coarse_occupancy(const uint8_t *__restrict__ bits, uint32_t C, uint32_t H, uint32_t *__restrict__ coarse) {
    const uint32_t Hc = H / 4, n = C * Hc * Hc * Hc, H3 = H * H * H;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t c = i / (Hc * Hc * Hc), r = i - c * Hc * Hc * Hc;
        const uint32_t cx = r / (Hc * Hc), cy = (r / Hc) % Hc, cz = r % Hc;
        // a 4-aligned 4x4x4 block is 64 consecutive Morton codes = 8 consecutive bytes
        const uint32_t m0 = morton3(cx * 4, cy * 4, cz * 4);
        const uint64_t v = *reinterpret_cast<const uint64_t *>(bits + ((size_t)c * H3 + m0) / 8);
        if (v) atomicOr(coarse + (i >> 5), 1u << (i & 31));
    }
}

// ---- sector-packed corner layout of a tiled grid (common.cuh: grid_lookup3q) ----
__global__ void k_pack_quads(GridMeta gm, const float2 *__restrict__ table, float4 *__restrict__ quads, uint32_t total) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        int l = 0;
#pragma unroll 1
        for (int k = 1; k < (int)gm.num_levels; ++k)
            if (i >= gm.offset[k]) l = k;
        const uint32_t q = i - gm.offset[l], m1 = gm.mul1[l];
        const float2 *tb = table + gm.offset[l];
        const float2 e0 = tb[grid_mod(gm, l, q)], e1 = tb[grid_mod(gm, l, q + 1)], e2 = tb[grid_mod(gm, l, q + m1)],
                     e3 = tb[grid_mod(gm, l, q + m1 + 1)];
        quads[2 * (size_t)i] = make_float4(e0.x, e0.y, e1.x, e1.y);
        quads[2 * (size_t)i + 1] = make_float4(e2.x, e2.y, e3.x, e3.y);
    }
}

// ---- fp16 oct layout of a tiled 3-D grid (common.cuh; read by lookup8o in head_tc_kernel.cu) ----
__global__ void k_pack_octs(GridMeta gm, const float2 *__restrict__ table, uint4 *__restrict__ octs, uint32_t total) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        int l = 0;
#pragma unroll 1
        for (int k = 1; k < (int)gm.num_levels; ++k)
            if (i >= gm.offset[k]) l = k;
        const uint32_t q = i - gm.offset[l], m1 = gm.mul1[l], m2 = gm.mul2[l];
        const float2 *tb = table + gm.offset[l];
        uint32_t w[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float2 e = tb[grid_mod(gm, l, q + (c & 1) + ((c & 2) ? m1 : 0u) + ((c & 4) ? m2 : 0u))];
            const __half2 h = __floats2half2_rn(e.x, e.y);
            w[c] = *reinterpret_cast<const uint32_t *>(&h);
        }
        octs[2 * (size_t)i] = make_uint4(w[0], w[1], w[2], w[3]);
        octs[2 * (size_t)i + 1] = make_uint4(w[4], w[5], w[6], w[7]);
    }
}

// 16-bit fixed-point octs (gather8.cuh OCT_I16): per-level step = max|T_l| / 32767, q = rn(T / step)
__global__ void k_level_absmax(GridMeta gm, const float2 *__restrict__ table, uint32_t total, uint32_t *__restrict__ amax_bits) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        int l = 0;
#pragma unroll 1
        for (int k = 1; k < (int)gm.num_levels; ++k)
            if (i >= gm.offset[k]) l = k;
        const float2 e = table[i];
        const float m = fmaxf(fabsf(e.x), fabsf(e.y));
        if (m > 0.f && !(m != m)) atomicMax(amax_bits + l, __float_as_uint(m));   // non-negative floats order like their bit patterns
    }
}
__global__ void k_level_step(const uint32_t *__restrict__ amax_bits, int n_levels, float *__restrict__ step) {
    const int l = threadIdx.x;
    if (l < n_levels) {
        const float m = __uint_as_float(amax_bits[l]);
        step[l] = m > 0.f ? m / 32767.0f : 1.0f;
    }
}
__global__ void k_pack_octs_i16(GridMeta gm, const float2 *__restrict__ table, uint4 *__restrict__ octs, uint32_t total,
                                const float *__restrict__ step) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        int l = 0;
#pragma unroll 1
        for (int k = 1; k < (int)gm.num_levels; ++k)
            if (i >= gm.offset[k]) l = k;
        const uint32_t q = i - gm.offset[l], m1 = gm.mul1[l], m2 = gm.mul2[l];
        const float2 *tb = table + gm.offset[l];
        const float inv = 1.0f / step[l];
        uint32_t w[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float2 e = tb[grid_mod(gm, l, q + (c & 1) + ((c & 2) ? m1 : 0u) + ((c & 4) ? m2 : 0u))];
            const int qx = max(-32767, min(32767, __float2int_rn(e.x * inv))), qy = max(-32767, min(32767, __float2int_rn(e.y * inv)));
            w[c] = ((uint32_t)qx & 0xFFFFu) | ((uint32_t)qy << 16);
        }
        octs[2 * (size_t)i] = make_uint4(w[0], w[1], w[2], w[3]);
        octs[2 * (size_t)i + 1] = make_uint4(w[4], w[5], w[6], w[7]);
    }
}

// ------------------------------------------------------------------------------------------------ launchers
// scratch: 16 uint32 (zeroed here); step: 16 floats
cudaError_t launch_pack_octs_i16(const GridMeta &gm, const float *table, void *octs, uint32_t total, uint32_t *scratch, float *step,
                                 cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(scratch, 0, 16 * sizeof(uint32_t), st);
    if (e != cudaSuccess) return e;
    k_level_absmax<<<grid_for(total, 256), 256, 0, st>>>(gm, (const float2 *)table, total, scratch);
    k_level_step<<<1, 32, 0, st>>>(scratch, (int)gm.num_levels, step);
    k_pack_octs_i16<<<grid_for(total, 256), 256, 0, st>>>(gm, (const float2 *)table, (uint4 *)octs, total, step);
    return cudaGetLastError();
}

cudaError_t launch_pack_octs(const GridMeta &gm, const float *table, void *octs, uint32_t total, cudaStream_t st) {
    k_pack_octs<<<grid_for(total, 256), 256, 0, st>>>(gm, (const float2 *)table, (uint4 *)octs, total);
    return cudaGetLastError();
}

cudaError_t launch_pack_quads(const GridMeta &gm, const float *table, float *quads, uint32_t total, cudaStream_t st) {
    k_pack_quads<<<grid_for(total, 256), 256, 0, st>>>(gm, (const float2 *)table, (float4 *)quads, total);
    return cudaGetLastError();
}

cudaError_t launch_coarse_occupancy(const uint8_t *bits, uint32_t C, uint32_t H, uint32_t *coarse, cudaStream_t st) {
    const uint32_t Hc = H / 4;
    k_coarse_occupancy<<<grid_for((uint64_t)C * Hc * Hc * Hc, 256), 256, 0, st>>>(bits, C, H, coarse);
    return cudaGetLastError();
}

cudaError_t launch_near_far(const float *rays_o, const float *rays_d, const float *aabb, uint32_t N, float min_near,
                            float *nears, float *fars, cudaStream_t st) {
    if (N == 0) return cudaSuccess;
    k_near_far<<<grid_for(N, 256), 256, 0, st>>>(rays_o, rays_d, aabb, N, min_near, nears, fars);
    return cudaGetLastError();
}

cudaError_t launch_march_rays(const MarchConst &mc, uint32_t n_alive, uint32_t n_step, const int32_t *rays_alive,
                              const float *rays_t, const float *rays_o, const float *rays_d, const float *fars,
                              float *xyzs, float *dirs, float *deltas, const float *noises, cudaStream_t st) {
    if (n_alive == 0) return cudaSuccess;
    k_march_rays<<<grid_for(n_alive, 128), 128, 0, st>>>(mc, n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, fars,
                                                          xyzs, dirs, deltas, noises);
    return cudaGetLastError();
}

cudaError_t launch_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t *rays_alive, float *rays_t,
                                  const float *sigmas, const float *rgbs, const float *deltas, float *weights_sum,
                                  float *depth, float *image, cudaStream_t st) {
    if (n_alive == 0) return cudaSuccess;
    k_composite_rays<<<grid_for(n_alive, 128), 128, 0, st>>>(n_alive, n_step, T_thresh, rays_alive, rays_t, sigmas, rgbs,
                                                              deltas, weights_sum, depth, image);
    return cudaGetLastError();
}

cudaError_t launch_grid_encode(const GridMeta &gm, const float *inputs, const float *table, float *outputs, uint32_t B,
                               cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    const uint32_t total = B * gm.num_levels;
    if (gm.dim == 3)
        k_grid_encode<3><<<grid_for(total, 256), 256, 0, st>>>(gm, inputs, (const float2 *)table, (float2 *)outputs, B);
    else
        k_grid_encode<2><<<grid_for(total, 256), 256, 0, st>>>(gm, inputs, (const float2 *)table, (float2 *)outputs, B);
    return cudaGetLastError();
}

cudaError_t launch_sh_encode(const float *inputs, float *outputs, uint32_t B, uint32_t degree, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    k_sh_encode<<<grid_for(B, 256), 256, 0, st>>>(inputs, outputs, B, degree);
    return cudaGetLastError();
}

cudaError_t launch_freq_encode(const float *inputs, uint32_t B, uint32_t D, uint32_t C, float *outputs, cudaStream_t st) {
    if (B * C == 0) return cudaSuccess;
    k_freq_encode<<<grid_for(B * C, 256), 256, 0, st>>>(inputs, B, D, C, outputs);
    return cudaGetLastError();
}

cudaError_t launch_occupancy_bounds(const uint8_t *bits, uint32_t n_bytes, uint32_t H3, int *bounds, cudaStream_t st) {
    k_occupancy_bounds<<<grid_for(n_bytes, 256), 256, 0, st>>>(bits, n_bytes, H3, bounds);
    return cudaGetLastError();
}

}  // namespace gfpp
