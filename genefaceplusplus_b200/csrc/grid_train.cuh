// grid_train.cuh -- the grid encoder's backward per (point, level), shared by the training fields (field_train_kernel.cu,
// torso_train_kernel.cu): the lookup's corners, weights and input derivative (gridencoder.cu:87-243), the table scatter
// (gridencoder.cu:246-340) and the input gradient through dy_dx.
#pragma once
#include "common.cuh"

namespace gfpp {

__device__ __forceinline__ float smoothstep_deriv(float x) { return 6.0f * x * (1.0f - x); }

template <int D>
__device__ __forceinline__ bool grid_cell(const GridMeta &gm, int l, const float *in, uint32_t (&pg)[3], float (&pos)[3], float (&deriv)[3]) {
#pragma unroll
    for (int d = 0; d < D; ++d)
        if (in[d] < 0.f || in[d] > 1.f) return false;
    const float sc = gm.scale[l];
    pg[2] = 0u; pos[2] = 0.f; deriv[2] = 1.f;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        float p = __fadd_rn(__fmul_rn(in[d], sc), gm.align_off);
        const float f0 = floorf(p);
        pg[d] = (uint32_t)f0;
        p -= f0;
        deriv[d] = 1.0f;
        if (gm.interp == 1) { deriv[d] = smoothstep_deriv(p); p = p * p * (3.0f - 2.0f * p); }
        pos[d] = p;
    }
    return true;
}

// table gradient of one (point, level): g scattered to the 2^D corners with vector reductions (gridencoder.cu:246-340)
template <int D>
__device__ __forceinline__ void grid_scatter(const GridMeta &gm, int l, const float *in, float2 g, float2 *__restrict__ grad_table) {
    uint32_t pg[3];
    float pos[3], deriv[3];
    if (!grid_cell<D>(gm, l, in, pg, pos, deriv)) return;
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
        atomicAdd(gt + grid_slot(gm, l, pl[0], pl[1], pl[2]), make_float2(w * g.x, w * g.y));
    }
}

// input gradient of one (point, level): gin[d] += g . dy_dx[d], dy_dx as the reference's forward computes it
template <int D>
__device__ __forceinline__ void grid_input_grad(const GridMeta &gm, const float2 *__restrict__ table, int l, const float *in, float2 g,
                                                float (&gin)[3]) {
    uint32_t pg[3];
    float pos[3], deriv[3];
    if (!grid_cell<D>(gm, l, in, pg, pos, deriv)) return;
    const float2 *tb = table + gm.offset[l];
    const float sc = gm.scale[l];
#pragma unroll
    for (int gd = 0; gd < D; ++gd) {
        float2 acc = make_float2(0.f, 0.f);
#pragma unroll
        for (int idx = 0; idx < (1 << (D - 1)); ++idx) {
            float w = sc;
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
        gin[gd] += g.x * acc.x;
        gin[gd] += g.y * acc.y;
    }
}

}  // namespace gfpp
