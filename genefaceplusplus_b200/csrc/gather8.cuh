// gather8.cuh -- consecutive levels (eight per call in lookup8) of a 3-D tiled grid for ONE sample out of the sector-packed "oct" tables
// (common.cuh: all eight corners of a cell in one 32-byte sector), shared by the tensor-core head kernels.
//
// Two oct formats:
//   OCT_F16  8 x half2: table values rounded to fp16, exactly what the reference does under autocast
//            (encoders/gridencoder/grid.py:43-44).
//   OCT_I16  8 x short2: 16-bit fixed point with ONE scale per level (value = q * step_l, step_l = max|T_l| / 32767):
//            absolute error <= step_l / 2, i.e. 2^-16 of the level's range instead of fp16's 2^-12 of each value -- the
//            "robust" precision mode uses it for the position grid, whose rounding error the ambient net amplifies
//            (tools/error_budget.py).  Decoded with one PRMT + one FADD per value (no conversion-pipe instruction).
// Interpolation is fp32 in both.  All N 256-bit loads of a call (N consecutive levels, eight in lookup8) are issued before the
// first is consumed; each level's arithmetic is the same whatever N is, so a level's value does not depend on how the levels of a
// sample are split into calls.
#pragma once
#include "common.cuh"

namespace gfpp {

enum OctFormat : int { OCT_F16 = 0, OCT_I16 = 1 };

// per-level metadata of one grid in SHARED memory, two 16-byte words per level:
//   {scale bits, mul1, mul2, offset}, {hmask, hsize, i16 step bits, 0}
__device__ __forceinline__ void stage_level_meta(const GridMeta &gm, const float *__restrict__ i16_step, uint4 *lvl, int tid) {
    if (tid < GFPP_MAX_LEVELS) {
        const bool on = (uint32_t)tid < gm.num_levels;
        const uint32_t st = (on && i16_step) ? __float_as_uint(i16_step[tid]) : 0u;
        lvl[2 * tid] = on ? make_uint4(__float_as_uint(gm.scale[tid]), gm.mul1[tid], gm.mul2[tid], gm.offset[tid]) : make_uint4(0, 0, 0, 0);
        lvl[2 * tid + 1] = on ? make_uint4(gm.hmask[tid], gm.hsize[tid], st, 0u) : make_uint4(0, 1u, 0, 0);
    }
}

// two int16 packed in a 32-bit word -> two floats, exact: 0x4B40'0000 | (q ^ 0x8000) is the float 12582912 + (q + 32768)
__device__ __forceinline__ float2 unpack_i16x2(uint32_t w) {
    const uint32_t b = w ^ 0x80008000u;
    const float lo = __uint_as_float(__byte_perm(b, 0x4B400000u, 0x7610));
    const float hi = __uint_as_float(__byte_perm(b, 0x4B400000u, 0x7632));
    return make_float2(lo - 12615680.0f, hi - 12615680.0f);   // 12582912 + 32768
}

// level j's cell at (u, v, w): returns the index of its oct in `octs` (uint4 pairs), and the position inside the cell in px, py, pz
__device__ __forceinline__ uint32_t oct_cell(const uint4 *lvl, int j, float align_off, float u, float v, float w, float &px, float &py,
                                             float &pz) {
    const uint4 m0 = lvl[2 * j], m1 = lvl[2 * j + 1];
    const float s = __uint_as_float(m0.x);
    px = __fadd_rn(__fmul_rn(u, s), align_off); py = __fadd_rn(__fmul_rn(v, s), align_off); pz = __fadd_rn(__fmul_rn(w, s), align_off);
    const float x0 = floorf(px), y0 = floorf(py), z0 = floorf(pz);
    px -= x0; py -= y0; pz -= z0;
    uint32_t q = (uint32_t)x0 + (uint32_t)y0 * m0.y + (uint32_t)z0 * m0.z;
    if (m1.x) q &= m1.x;                 // grid_mod (common.cuh)
    else if (q >= m1.y) q %= m1.y;
    return m0.w + q;
}

// the octs of N consecutive levels at (u, v, w) towards L2, without holding a register for their data
template <int N>
__device__ __forceinline__ void prefetch_levels_l2(const uint4 *lvl, float align_off, const uint4 *__restrict__ octs, float u, float v, float w) {
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
        float px, py, pz;
        const uint32_t o = oct_cell(lvl, j, align_off, u, v, w, px, py, pz);
        asm volatile("prefetch.global.L2 [%0];" ::"l"(octs + 2 * (size_t)o));
    }
}

template <int FMT, bool SMOOTH, int N>
__device__ __forceinline__ void lookup_impl(const uint4 *lvl, float align_off, const uint4 *__restrict__ octs, float u, float v, float w,
                                            float (&f)[2 * N]) {
    float fx[N], fy[N], fz[N];
    uint4 lo4[N], hi4[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
        float px, py, pz;
        const uint32_t o = oct_cell(lvl, j, align_off, u, v, w, px, py, pz);
        if (SMOOTH) {
            px = px * px * (3.0f - 2.0f * px);
            py = py * py * (3.0f - 2.0f * py);
            pz = pz * pz * (3.0f - 2.0f * pz);
        }
        fx[j] = px; fy[j] = py; fz[j] = pz;
        ldg256_na(octs + 2 * (size_t)o, lo4[j], hi4[j]);   // the whole 32-byte oct in one request
    }
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const uint32_t c[8] = {lo4[j].x, lo4[j].y, lo4[j].z, lo4[j].w, hi4[j].x, hi4[j].y, hi4[j].z, hi4[j].w};
        const float wx[2] = {1.0f - fx[j], fx[j]}, wy[2] = {1.0f - fy[j], fy[j]}, wz[2] = {1.0f - fz[j], fz[j]};
        const float wyz[4] = {wy[0] * wz[0], wy[1] * wz[0], wy[0] * wz[1], wy[1] * wz[1]};
        float ax = 0.f, ay = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float2 e = FMT == OCT_I16 ? unpack_i16x2(c[i]) : __half22float2(*reinterpret_cast<const __half2 *>(&c[i]));
            const float wgt = wx[i & 1] * wyz[i >> 1];
            ax += wgt * e.x;
            ay += wgt * e.y;
        }
        if (FMT == OCT_I16) {
            const float step = __uint_as_float(lvl[2 * j + 1].z);
            ax *= step; ay *= step;
        }
        f[2 * j] = ax;
        f[2 * j + 1] = ay;
    }
    if (u < 0.f || u > 1.f || v < 0.f || v > 1.f || w < 0.f || w > 1.f) {   // outside the grid: zeros (gridencoder.cu:108-118)
#pragma unroll
        for (int i = 0; i < 2 * N; ++i) f[i] = 0.f;
    }
}

// N consecutive levels, starting at the level whose metadata `lvl` points at
template <int FMT, int N>
__device__ __forceinline__ void lookup_levels(const uint4 *lvl, float align_off, bool smooth, const uint4 *__restrict__ octs, float u, float v,
                                              float w, float (&f)[2 * N]) {
    if (smooth) lookup_impl<FMT, true, N>(lvl, align_off, octs, u, v, w, f);   // warp-uniform: only one instantiation ever runs (I-cache)
    else lookup_impl<FMT, false, N>(lvl, align_off, octs, u, v, w, f);
}

template <int FMT>
__device__ __forceinline__ void lookup8(const uint4 *lvl, float align_off, bool smooth, const uint4 *__restrict__ octs, float u, float v, float w,
                                        float (&f)[16]) {
    lookup_levels<FMT, 8>(lvl, align_off, smooth, octs, u, v, w, f);
}

}  // namespace gfpp
