// torso_common.cuh -- device helpers shared by the torso kernels (torso_kernel.cu: radnerf_torso.py field; torso_sr_kernel.cu:
// radnerf_torso_sr.py field; the grid query and the training fields): frequency-encoder entries, small FFMA tile GEMMs out of
// shared memory (all of them but k_epilogue, which runs its MLPs on the tensor cores), grid_sample restated.
#pragma once
#include "common.cuh"

namespace gfpp {
namespace torsoc {

// freq-encoder entry c of a D-dim input (freqencoder.cu:47-57); accurate sinf
__device__ __forceinline__ float freq_entry(const float *x, int D, int c) {
    if (c < D) return x[c];
    const int col = c / D - 1, d = c % D, f = col / 2;
    return sinf(__fadd_rn(scalbnf(x[d], f), (float)(col % 2) * (3.141592653589793f / 2)));
}

// LeakyReLU(0.02) of the torso-SR model's head-aware encoder
__device__ __forceinline__ float leaky002(float x) { return x > 0.f ? x : 0.02f * x; }

// acc[i][j] += A[row_i][k] * W[k][col_j], rows ty*4+i / 64+ty*4+(i-4), cols tx*NC+j; W is [K][N], N = 16*NC
template <int NC, int K, int LDT>
__device__ __forceinline__ void small_gemm(float (&acc)[8][NC], const float *__restrict__ sA, const float *__restrict__ sW,
                                           int ty, int tx) {
    constexpr int N = 16 * NC;
    const float *a0 = sA + (ty * 4) * LDT, *a1 = sA + (64 + ty * 4) * LDT;
#pragma unroll 2
    for (int k4 = 0; k4 < K; k4 += 4) {
        float4 av[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            av[i] = *reinterpret_cast<const float4 *>(a0 + i * LDT + k4);
            av[4 + i] = *reinterpret_cast<const float4 *>(a1 + i * LDT + k4);
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            float b[NC];
#pragma unroll
            for (int j = 0; j < NC; ++j) b[j] = sW[(k4 + kk) * N + tx * NC + j];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float ai = kk == 0 ? av[i].x : kk == 1 ? av[i].y : kk == 2 ? av[i].z : av[i].w;
#pragma unroll
                for (int j = 0; j < NC; ++j) acc[i][j] = fmaf(ai, b[j], acc[i][j]);
            }
        }
    }
}

template <int NC, int LDT>
__device__ __forceinline__ void store_relu(const float (&acc)[8][NC], float *sA, const float *bias, int ty, int tx) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4);
#pragma unroll
        for (int j = 0; j < NC; ++j) {
            const int c = tx * NC + j;
            sA[row * LDT + c] = fmaxf(acc[i][j] + (bias ? __ldg(bias + c) : 0.f), 0.f);
        }
    }
}

// F.grid_sample(grid[1,1,G,G], coords, align_corners=True, bilinear, zeros padding) at one point
// (ATen grid_sampler_2d: unnormalise ((c+1)/2)*(size-1); weights nw,ne,sw,se in that order).  ATen's CUDA kernel accumulates with
// `out += v * w`, which nvcc contracts to an FMA: kFma = true restates that exactly on any grid (the training mask, gfpp_torso_mask);
// the default rounds each product, which is the same wherever v * w is exact -- a 0 / 1 grid -- and is what the render epilogues use.
template <bool kFma = false>
__device__ __forceinline__ float sample_density(const float *__restrict__ grid, int G, float cx, float cy) {
    const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(cx, 1.0f), 2.0f), (float)(G - 1));
    const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(cy, 1.0f), 2.0f), (float)(G - 1));
    const float x0 = floorf(ix), y0 = floorf(iy);
    const float x1 = x0 + 1.0f, y1 = y0 + 1.0f;
    const float nw = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(y1, iy)), ne = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(y1, iy));
    const float sw = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(iy, y0)), se = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(iy, y0));
    const int ix0 = (int)x0, iy0 = (int)y0, ix1 = ix0 + 1, iy1 = iy0 + 1;
    auto at = [&](int yy, int xx) -> float { return (xx >= 0 && xx < G && yy >= 0 && yy < G) ? __ldg(grid + yy * G + xx) : 0.0f; };
    auto acc = [](float o, float v, float w) { return kFma ? __fmaf_rn(v, w, o) : __fadd_rn(o, __fmul_rn(v, w)); };
    float out = 0.f;
    out = acc(out, at(iy0, ix0), nw);
    out = acc(out, at(iy0, ix1), ne);
    out = acc(out, at(iy1, ix0), sw);
    out = acc(out, at(iy1, ix1), se);
    return out;
}


}  // namespace torsoc
}  // namespace gfpp
