// grid_half_kernels.cu -- the multi-resolution grid encoder on half tables (gfpp.h section (L)): what the reference's
// scalar_t = at::Half instantiations of kernel_grid, kernel_grid_backward and kernel_input_backward compute
// (gridencoder.cu:87-368) when autocast hands it a half table (grid.py:41-44), for C = 2 and D in {2, 3}.
//
// at::Half arithmetic, restated site by site (c10 Half: every operator converts to fp32, computes, and rounds back):
//   results[ch] += w * grid[i]     the fp32 product w * g is rounded to half, the sum of two halves formed in fp32 and rounded
//   grid[r] - grid[l]              rounded to half before the fp32 products with w and pos_deriv
//   (__half)(w * grad[c])          the table-gradient term, rounded to half, then one f16x2 reduction per corner
//   result += grad * dy_dx         half product, half sum
// Every rounding is round-to-nearest-even (__float2half_rn), as c10::Half(float) is.  The level constants come from the device
// exp2f exactly as the reference kernel derives them (scale = exp2f(level * S) * H - 1, resolution = ceil(scale) + 1) -- unlike
// the fp32 ops, which take them from the host (capi.cu: fill_grid_meta) -- so that these kernels are bit-exact against the
// reference's own half kernels.  FMA contraction follows the reference's SASS (cuobjdump -sass of its sm_90a build): it forms two
// FFMAs, scale = fma(exp2f(level * S), H, -1) and pos = fma(x, scale, 0.5); smoothstep is (p * p) * (3 - (p + p)) and every
// product and sum of the running sums rounds on its own.  Both are written here with explicit intrinsics, so that nvcc cannot
// contract differently.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "grid_half.cuh"

namespace gfpp {

namespace {

__device__ __forceinline__ __half f2h(float f) { return __float2half_rn(f); }
__device__ __forceinline__ float h2f(__half h) { return __half2float(h); }
// at::Half += float (gridencoder.cu:186, 234): the addend is rounded to half first
__device__ __forceinline__ __half hacc(__half acc, float t) { return f2h(__fadd_rn(h2f(acc), h2f(f2h(t)))); }

struct Level {
    float scale;
    uint32_t res, hs;
};

__device__ __forceinline__ Level level_of(const HalfGridArgs &g, uint32_t level) {
    Level v;
    v.hs = g.offset[level + 1] - g.offset[level];
    v.scale = __fmaf_rn(exp2f((float)level * g.S), (float)g.H, -1.0f);    // gridencoder.cu:138: device exp2f, contracted as in its SASS
    v.res = (uint32_t)ceilf(v.scale) + 1;
    return v;
}

// get_grid_index (gridencoder.cu:66-84) in half2 slots
template <int D>
__device__ __forceinline__ uint32_t slot_of(const HalfGridArgs &g, const Level &lv, const uint32_t (&p)[D]) {
    uint32_t stride = 1, index = 0;
#pragma unroll
    for (int d = 0; d < D && stride <= lv.hs; ++d) {
        index += p[d] * stride;
        stride *= g.align_corners ? lv.res : lv.res + 1;
    }
    if (g.gridtype == 0 && stride > lv.hs) {
        constexpr uint32_t primes[3] = {1u, 2654435761u, 805459861u};
        index = 0;
#pragma unroll
        for (int d = 0; d < D; ++d) index ^= p[d] * primes[d];
    }
    return index % lv.hs;
}

// cell, fractional position (smoothstep applied) and its derivative (gridencoder.cu:146-158)
template <int D>
__device__ __forceinline__ void cell_of(const HalfGridArgs &g, const Level &lv, const float (&in)[D], uint32_t (&pg)[D],
                                        float (&pos)[D], float (&deriv)[D]) {
    const float off = g.align_corners ? 0.0f : 0.5f;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        float p = __fmaf_rn(in[d], lv.scale, off);
        pg[d] = (uint32_t)floorf(p);
        p = __fsub_rn(p, (float)pg[d]);
        if (g.interp == 1) {
            deriv[d] = __fmul_rn(__fmul_rn(6.0f, p), __fsub_rn(1.0f, p));
            p = __fmul_rn(__fmul_rn(p, p), __fsub_rn(3.0f, __fmul_rn(2.0f, p)));   // 2p is exact (SASS: p + p)
        } else {
            deriv[d] = 1.0f;
        }
        pos[d] = p;
    }
}

template <int D>
__device__ __forceinline__ bool load_inputs(const float *__restrict__ inputs, uint32_t b, float (&in)[D]) {
    bool oob = false;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        in[d] = inputs[(size_t)b * D + d];
        if (in[d] < 0.f || in[d] > 1.f) oob = true;
    }
    return oob;
}

// f16x2 vector reduction, no flush to zero: what atomicAdd(__half2 *, __half2) compiles to when its result is unused
__device__ __forceinline__ void red_f16x2(__half2 *addr, __half2 v) {
    asm volatile("red.global.add.noftz.f16x2 [%0], %1;" ::"l"(addr), "r"(*reinterpret_cast<uint32_t *>(&v)) : "memory");
}

// forward: outputs [L,B] half2, dy_dx [B,L,D] half2 or null (gridencoder.cu:87-244); one thread per (point, level)
template <int D>
__global__ void __launch_bounds__(512) k_grid_half_fwd(const HalfGridArgs g, const float *__restrict__ inputs,
                                                       const __half2 *__restrict__ table, __half2 *__restrict__ outputs,
                                                       __half2 *__restrict__ dy_dx, uint32_t B) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    const __half2 zero = __float2half2_rn(0.f);
    float in[D];
    __half2 *dd = dy_dx ? dy_dx + ((size_t)b * g.L + level) * D : nullptr;
    if (load_inputs<D>(inputs, b, in)) {
        outputs[(size_t)level * B + b] = zero;
        if (dd) {
#pragma unroll
            for (int d = 0; d < D; ++d) dd[d] = zero;
        }
        return;
    }
    const Level lv = level_of(g, level);
    const __half2 *tb = table + g.offset[level];
    uint32_t pg[D];
    float pos[D], deriv[D];
    cell_of<D>(g, lv, in, pg, pos, deriv);

    __half r0 = __float2half_rn(0.f), r1 = r0;
#pragma unroll
    for (int idx = 0; idx < (1 << D); ++idx) {
        float w = 1.0f;
        uint32_t pl[D];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            if ((idx & (1 << d)) == 0) { w = __fmul_rn(w, __fsub_rn(1.0f, pos[d])); pl[d] = pg[d]; }
            else { w = __fmul_rn(w, pos[d]); pl[d] = pg[d] + 1; }
        }
        const __half2 v = __ldg(tb + slot_of<D>(g, lv, pl));
        r0 = hacc(r0, __fmul_rn(w, __low2float(v)));
        r1 = hacc(r1, __fmul_rn(w, __high2float(v)));
    }
    outputs[(size_t)level * B + b] = __halves2half2(r0, r1);
    if (!dd) return;

#pragma unroll
    for (int gd = 0; gd < D; ++gd) {
        __half a0 = __float2half_rn(0.f), a1 = a0;
#pragma unroll
        for (int idx = 0; idx < (1 << (D - 1)); ++idx) {
            float w = lv.scale;
            uint32_t pl[D];
#pragma unroll
            for (int nd = 0; nd < D - 1; ++nd) {
                const int d = nd >= gd ? nd + 1 : nd;
                if ((idx & (1 << nd)) == 0) { w = __fmul_rn(w, __fsub_rn(1.0f, pos[d])); pl[d] = pg[d]; }
                else { w = __fmul_rn(w, pos[d]); pl[d] = pg[d] + 1; }
            }
            pl[gd] = pg[gd];
            const __half2 lft = __ldg(tb + slot_of<D>(g, lv, pl));
            pl[gd] = pg[gd] + 1;
            const __half2 rgt = __ldg(tb + slot_of<D>(g, lv, pl));
            // (grid[r] - grid[l]) is an at::Half difference: rounded before the fp32 products
            const float d0 = h2f(f2h(__fsub_rn(__low2float(rgt), __low2float(lft))));
            const float d1 = h2f(f2h(__fsub_rn(__high2float(rgt), __high2float(lft))));
            a0 = hacc(a0, __fmul_rn(__fmul_rn(w, d0), deriv[gd]));
            a1 = hacc(a1, __fmul_rn(__fmul_rn(w, d1), deriv[gd]));
        }
        dd[gd] = __halves2half2(a0, a1);
    }
}

// table gradient (gridencoder.cu:246-340): one thread per (point, level), one f16x2 reduction per corner
template <int D>
__global__ void __launch_bounds__(256) k_grid_half_bwd(const HalfGridArgs g, const __half2 *__restrict__ grad,
                                                       const float *__restrict__ inputs, __half2 *__restrict__ grad_table, uint32_t B) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    float in[D];
    if (load_inputs<D>(inputs, b, in)) return;   // grad_embeddings is zero-initialised by the caller (grid.py:76)
    const Level lv = level_of(g, level);
    uint32_t pg[D];
    float pos[D], deriv[D];
    cell_of<D>(g, lv, in, pg, pos, deriv);
    const __half2 gc = grad[(size_t)level * B + b];
    const float g0 = __low2float(gc), g1 = __high2float(gc);
    __half2 *gt = grad_table + g.offset[level];
#pragma unroll
    for (int idx = 0; idx < (1 << D); ++idx) {
        float w = 1.0f;
        uint32_t pl[D];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            if ((idx & (1 << d)) == 0) { w = __fmul_rn(w, __fsub_rn(1.0f, pos[d])); pl[d] = pg[d]; }
            else { w = __fmul_rn(w, pos[d]); pl[d] = pg[d] + 1; }
        }
        red_f16x2(gt + slot_of<D>(g, lv, pl), __halves2half2(f2h(__fmul_rn(w, g0)), f2h(__fmul_rn(w, g1))));
    }
}

// input gradient (gridencoder.cu:343-368): grad_inputs[b,d] = sum over (level, channel) of grad * dy_dx, half products, half sum
template <int D>
__global__ void __launch_bounds__(256) k_grid_half_input_bwd(const __half *__restrict__ grad, const __half *__restrict__ dy_dx,
                                                             __half *__restrict__ grad_inputs, uint32_t B, uint32_t L) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * D) return;
    const uint32_t b = t / D, d = t - b * D;
    const __half *dd = dy_dx + (size_t)b * L * D * 2;
    __half r = __float2half_rn(0.f);
    for (uint32_t l = 0; l < L; ++l) {
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
            const __half p = f2h(__fmul_rn(h2f(grad[((size_t)l * B + b) * 2 + ch]), h2f(dd[(l * D + d) * 2 + ch])));
            r = f2h(__fadd_rn(h2f(r), h2f(p)));
        }
    }
    grad_inputs[t] = r;
}

inline uint32_t blocks_for(uint32_t n, uint32_t threads) { return (n + threads - 1) / threads; }

}  // namespace

cudaError_t launch_grid_half_forward(const HalfGridArgs &g, uint32_t D, const float *inputs, const void *table, void *outputs, void *dy_dx,
                                     uint32_t B, cudaStream_t st) {
    const dim3 grid(blocks_for(B, 512), g.L);
    if (D == 3)
        k_grid_half_fwd<3><<<grid, 512, 0, st>>>(g, inputs, (const __half2 *)table, (__half2 *)outputs, (__half2 *)dy_dx, B);
    else
        k_grid_half_fwd<2><<<grid, 512, 0, st>>>(g, inputs, (const __half2 *)table, (__half2 *)outputs, (__half2 *)dy_dx, B);
    return cudaGetLastError();
}

cudaError_t launch_grid_half_backward(const HalfGridArgs &g, uint32_t D, const void *grad, const float *inputs, void *grad_table,
                                      const void *dy_dx, void *grad_inputs, uint32_t B, int *launches, cudaStream_t st) {
    const dim3 grid(blocks_for(B, 256), g.L);
    if (D == 3) k_grid_half_bwd<3><<<grid, 256, 0, st>>>(g, (const __half2 *)grad, inputs, (__half2 *)grad_table, B);
    else k_grid_half_bwd<2><<<grid, 256, 0, st>>>(g, (const __half2 *)grad, inputs, (__half2 *)grad_table, B);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    *launches = 1;
    if (!dy_dx) return cudaSuccess;
    const uint32_t n = B * D;
    if (D == 3)
        k_grid_half_input_bwd<3><<<blocks_for(n, 256), 256, 0, st>>>((const __half *)grad, (const __half *)dy_dx, (__half *)grad_inputs, B, g.L);
    else
        k_grid_half_input_bwd<2><<<blocks_for(n, 256), 256, 0, st>>>((const __half *)grad, (const __half *)dy_dx, (__half *)grad_inputs, B, g.L);
    e = cudaGetLastError();
    if (e == cudaSuccess) *launches = 2;
    return e;
}

}  // namespace gfpp
