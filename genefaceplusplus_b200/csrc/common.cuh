// common.cuh -- shared device helpers of libgfpp (sm_90a).
//
// The ray-march helpers make DISCRETE decisions (cell index, occupancy bit, "t < far"), so their fp32
// arithmetic is written with explicit round-to-nearest intrinsics (no FMA contraction) in exactly the
// evaluation order of the reference kernel (modules/radnerfs/raymarching/src/raymarching.cu:857-927,
// helpers :19-81) and of its CPU restatement oracle/native_ops.c.  See SURVEY.md section 7, H2.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#define GFPP_MAX_LEVELS 16

namespace gfpp {

__device__ __forceinline__ float clampf(float v, float lo, float hi) { return fminf(hi, fmaxf(lo, v)); }

// 10-bit-per-axis Morton interleave (raymarching.cu:57-72)
__device__ __forceinline__ uint32_t spread3(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
__device__ __forceinline__ uint32_t morton3(uint32_t x, uint32_t y, uint32_t z) {
    return spread3(x) | (spread3(y) << 1) | (spread3(z) << 2);
}

// ---------------------------------------------------------------------------------------------
// Marching constants shared by the per-op kernel and the fused renderer.
struct MarchConst {
    float bound, dt_gamma, dt_min, dt_max, rH, H3, Hm1, fC, fH;
    uint32_t C, H;
    const uint8_t *bits;
    // tight cell-space bounds of the occupied voxels of cascade 0..C-1 (inclusive); cells outside are
    // known empty, so their bit need not be read.  lo > hi means "no bounds available: always read".
    int bb_lo[3], bb_hi[3];
    // optional coarse occupancy: bit (level*Hc^3 + (cx*Hc + cy)*Hc + cz) is the OR of the 4x4x4 fine cells of coarse
    // cell (cx,cy,cz); a clear bit proves the fine cell empty without touching the fine bitfield (nullptr: unused).
    const uint32_t *coarse;
    uint32_t Hc;
};

__host__ __device__ inline void march_const_init(MarchConst &mc, float bound, float dt_gamma, uint32_t max_steps,
                                                 uint32_t C, uint32_t H, const uint8_t *bits) {
    mc.bound = bound;
    mc.dt_gamma = dt_gamma;
    const float sqrt3 = 1.7320508075688772f;
    // raymarching.cu:866-867
    mc.dt_max = 2 * sqrt3 * (float)(1 << (C - 1)) / (float)H;
    mc.dt_min = fminf(mc.dt_max, 2 * sqrt3 / (float)max_steps);
    mc.rH = 1.0f / (float)H;
    mc.H3 = (float)(H * H * H);
    mc.Hm1 = (float)(H - 1);
    mc.fC = (float)C;
    mc.fH = (float)H;
    mc.C = C;
    mc.H = H;
    mc.bits = bits;
    mc.bb_lo[0] = mc.bb_lo[1] = mc.bb_lo[2] = 1;
    mc.bb_hi[0] = mc.bb_hi[1] = mc.bb_hi[2] = 0;
    mc.coarse = nullptr;
    mc.Hc = H / 4;
}

struct RayGeom {
    float ox, oy, oz, dx, dy, dz, rdx, rdy, rdz;
};

__device__ __forceinline__ void ray_geom_init(RayGeom &g, float ox, float oy, float oz, float dx, float dy, float dz) {
    g.ox = ox; g.oy = oy; g.oz = oz;
    g.dx = dx; g.dy = dy; g.dz = dz;
    g.rdx = __fdiv_rn(1.0f, dx);
    g.rdy = __fdiv_rn(1.0f, dy);
    g.rdz = __fdiv_rn(1.0f, dz);
}

// slab test (raymarching.cu:91-145).  Returns near/far; a miss sets both to FLT_MAX.
__device__ __forceinline__ void near_far(const RayGeom &g, const float *aabb, float min_near, float &near, float &far) {
    float tn = __fmul_rn(__fsub_rn(aabb[0], g.ox), g.rdx), tf = __fmul_rn(__fsub_rn(aabb[3], g.ox), g.rdx);
    if (tn > tf) { float s = tn; tn = tf; tf = s; }
    float tny = __fmul_rn(__fsub_rn(aabb[1], g.oy), g.rdy), tfy = __fmul_rn(__fsub_rn(aabb[4], g.oy), g.rdy);
    if (tny > tfy) { float s = tny; tny = tfy; tfy = s; }
    if (tn > tfy || tny > tf) { near = far = FLT_MAX; return; }
    if (tny > tn) tn = tny;
    if (tfy < tf) tf = tfy;
    float tnz = __fmul_rn(__fsub_rn(aabb[2], g.oz), g.rdz), tfz = __fmul_rn(__fsub_rn(aabb[5], g.oz), g.rdz);
    if (tnz > tfz) { float s = tnz; tnz = tfz; tfz = s; }
    if (tn > tfz || tnz > tf) { near = far = FLT_MAX; return; }
    if (tnz > tn) tn = tnz;
    if (tfz < tf) tf = tfz;
    if (tn < min_near) tn = min_near;
    near = tn;
    far = tf;
}

__device__ __forceinline__ float step_len(const MarchConst &mc, float t) {
    return clampf(__fmul_rn(t, mc.dt_gamma), mc.dt_min, mc.dt_max);
}

// cell coordinate along one axis: (int)clamp(0.5 * (p * rb + 1) * H, 0, H-1) with the product taken in
// DOUBLE because of the reference's 0.5 literal (raymarching.cu:890-892).  When H is a power of two the double
// product 0.5*u*H is exactly the float product u*(H/2) (scaling by a power of two is exact), so the fp64 pipe is
// only used for odd grid sizes.
__device__ __forceinline__ int cell_of(float p, float mip_rbound, const MarchConst &mc) {
    const float u = __fadd_rn(__fmul_rn(p, mip_rbound), 1.0f);
    float c;
    if ((mc.H & (mc.H - 1)) == 0) c = __fmul_rn(u, 0.5f * mc.fH);
    else c = __double2float_rn(__dmul_rn(__dmul_rn(0.5, (double)u), (double)mc.H));
    return (int)clampf(c, 0.0f, mc.Hm1);
}

// Loop-invariant pieces of the marcher (single cascade: the mip level is always 0, raymarching.cu:881-886).
struct MarchHoist {
    bool single, have_bb;
    float mip_bound, mip_rbound, sx, sy, sz;
};
__device__ __forceinline__ void march_hoist(const MarchConst &mc, const RayGeom &g, MarchHoist &h) {
    h.single = mc.C == 1;
    h.mip_bound = fminf(1.0f, mc.bound);
    h.mip_rbound = __fdiv_rn(1.0f, h.mip_bound);
    h.sx = copysignf(1.0f, g.dx); h.sy = copysignf(1.0f, g.dy); h.sz = copysignf(1.0f, g.dz);
    h.have_bb = mc.bb_lo[0] <= mc.bb_hi[0];
}

// One iteration of the reference loop (raymarching.cu:873-927) at parameter t (< far).  Occupied cell: returns true with
// the sample (x,y,z,dt) and t UNCHANGED.  Empty cell: advances t past the voxel and returns false.  `cost` is incremented
// by 4 when the fine bitfield had to be read and by 1 otherwise (used to bound per-round prefetch work).
__device__ __forceinline__ bool march_cell(const MarchConst &mc, const RayGeom &g, const MarchHoist &h, float &t, float &x, float &y,
                                           float &z, float &dt, int &cost) {
    x = clampf(__fadd_rn(g.ox, __fmul_rn(t, g.dx)), -mc.bound, mc.bound);
    y = clampf(__fadd_rn(g.oy, __fmul_rn(t, g.dy)), -mc.bound, mc.bound);
    z = clampf(__fadd_rn(g.oz, __fmul_rn(t, g.dz)), -mc.bound, mc.bound);
    dt = step_len(mc, t);
    int level = 0;
    float mip_bound = h.mip_bound, mip_rbound = h.mip_rbound;
    if (!h.single) {
        int e1, e2;
        (void)frexpf(fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z))), &e1);
        // mip_from_dt: dt * H in float, then * 0.5 in double, rounded to float (raymarching.cu:50)
        (void)frexpf(__double2float_rn(__dmul_rn((double)__fmul_rn(dt, mc.fH), 0.5)), &e2);
        const int l1 = (int)fminf(mc.fC - 1.0f, fmaxf(0.0f, (float)e1));
        const int l2 = (int)fminf(mc.fC - 1.0f, fmaxf(0.0f, (float)e2));
        level = max(l1, l2);
        mip_bound = fminf(scalbnf(1.0f, level), mc.bound);
        mip_rbound = __fdiv_rn(1.0f, mip_bound);
    }
    const int nx = cell_of(x, mip_rbound, mc), ny = cell_of(y, mip_rbound, mc), nz = cell_of(z, mip_rbound, mc);
    bool occ = false;
    bool known_empty = h.have_bb && (nx < mc.bb_lo[0] || nx > mc.bb_hi[0] || ny < mc.bb_lo[1] || ny > mc.bb_hi[1] ||
                                     nz < mc.bb_lo[2] || nz > mc.bb_hi[2]);
    if (!known_empty && mc.coarse) {
        const uint32_t ci = (uint32_t)level * mc.Hc * mc.Hc * mc.Hc + (((uint32_t)nx >> 2) * mc.Hc + ((uint32_t)ny >> 2)) * mc.Hc + ((uint32_t)nz >> 2);
        known_empty = ((mc.coarse[ci >> 5] >> (ci & 31)) & 1u) == 0u;
    }
    if (!known_empty) {
        // bit index formed in float (raymarching.cu:894): exact while below 2^24
        const uint32_t bit = (uint32_t)__fadd_rn(__fmul_rn((float)level, mc.H3),
                                                 (float)morton3((uint32_t)nx, (uint32_t)ny, (uint32_t)nz));
        occ = (__ldg(mc.bits + (bit >> 3)) >> (bit & 7)) & 1;
        cost += 4;
    } else {
        cost += 1;
    }
    if (occ) return true;
    // distance to the far face of this voxel along the ray (raymarching.cu:916-919)
    const float fx = __fadd_rn(__fadd_rn((float)nx, 0.5f), __fmul_rn(0.5f, h.sx));
    const float fy = __fadd_rn(__fadd_rn((float)ny, 0.5f), __fmul_rn(0.5f, h.sy));
    const float fz = __fadd_rn(__fadd_rn((float)nz, 0.5f), __fmul_rn(0.5f, h.sz));
    const float tx = __fmul_rn(__fsub_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fmul_rn(fx, mc.rH), 2.0f), 1.0f), mip_bound), x), g.rdx);
    const float ty = __fmul_rn(__fsub_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fmul_rn(fy, mc.rH), 2.0f), 1.0f), mip_bound), y), g.rdy);
    const float tz = __fmul_rn(__fsub_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fmul_rn(fz, mc.rH), 2.0f), 1.0f), mip_bound), z), g.rdz);
    const float tt = __fadd_rn(t, fmaxf(0.0f, fminf(tx, fminf(ty, tz))));
    do {
        t = __fadd_rn(t, step_len(mc, t));
    } while (t < tt);
    return false;
}

// Advance `t` to the next occupied sample on the ray.  On success returns true with the sample
// position (x,y,z), its step dt, and t already advanced PAST the sample (t += dt), exactly like one
// "occupied" iteration of the reference loop.  Returns false when t >= far (ray exhausted).
__device__ __forceinline__ bool march_next(const MarchConst &mc, const RayGeom &g, float far, float &t, float &x,
                                           float &y, float &z, float &dt) {
    MarchHoist h;
    march_hoist(mc, g, h);
    int cost = 0;
    while (t < far) {
        if (march_cell(mc, g, h, t, x, y, z, dt, cost)) {
            t = __fadd_rn(t, dt);
            return true;
        }
    }
    return false;
}

// Resumable variant for prefetching: runs until a sample is found (returns 1, t = the sample's PRE-step parameter),
// the ray is exhausted (0) or `budget` cost units are spent (2, t = resume point).  Splitting the loop across calls is
// exact because every iteration is a pure function of t.
__device__ __forceinline__ int march_budget(const MarchConst &mc, const RayGeom &g, float far, float &t, int &budget) {
    MarchHoist h;
    march_hoist(mc, g, h);
    float x, y, z, dt;
    while (t < far) {
        if (budget <= 0) return 2;
        int cost = 0;
        const bool occ = march_cell(mc, g, h, t, x, y, z, dt, cost);
        budget -= cost;
        if (occ) return 1;
    }
    return 0;
}

// The emit step of the reference loop for a sample known to sit at parameter t_pre: position, step, t advanced past it.
__device__ __forceinline__ void sample_at(const MarchConst &mc, const RayGeom &g, float t_pre, float &t, float &x, float &y,
                                          float &z, float &dt) {
    x = clampf(__fadd_rn(g.ox, __fmul_rn(t_pre, g.dx)), -mc.bound, mc.bound);
    y = clampf(__fadd_rn(g.oy, __fmul_rn(t_pre, g.dy)), -mc.bound, mc.bound);
    z = clampf(__fadd_rn(g.oz, __fmul_rn(t_pre, g.dz)), -mc.bound, mc.bound);
    dt = step_len(mc, t_pre);
    t = __fadd_rn(t_pre, dt);
}

// ---------------------------------------------------------------------------------------------
// Multi-resolution grid (gridencoder.cu:50-84, 87-196).  Level constants are precomputed on the host
// with the same libm calls the oracle uses (exp2f, ceil) -- see capi.cu: fill_grid_meta().
struct GridMeta {
    float scale[GFPP_MAX_LEVELS];      // exp2f(l*S)*H - 1
    uint32_t offset[GFPP_MAX_LEVELS];  // table offset in entries
    uint32_t hsize[GFPP_MAX_LEVELS];   // entries in the level
    uint32_t mul1[GFPP_MAX_LEVELS];    // stride of dim 1 (0 if the dim is dropped: get_grid_index quirk, H5)
    uint32_t mul2[GFPP_MAX_LEVELS];    // stride of dim 2 (0 if dropped)
    uint32_t hashed[GFPP_MAX_LEVELS];  // 1 if gridtype==hash and the level overflows its table
    uint32_t hmask[GFPP_MAX_LEVELS];   // hsize-1 when hsize is a power of two (index % hsize == index & hmask), else 0
    uint32_t num_levels, dim, interp;
    float align_off;                   // 0.5 unless align_corners
    uint32_t quad_ok;                  // 1: the sector-packed corner layout (see grid_lookup3q) is valid for this grid
};

// table slot of integer cell (x,y,z) in level l: get_grid_index (gridencoder.cu:66-84)
__device__ __forceinline__ uint32_t grid_slot(const GridMeta &gm, int l, uint32_t x, uint32_t y, uint32_t z) {
    uint32_t idx;
    if (gm.hashed[l]) {
        idx = (x * 1u) ^ (y * 2654435761u) ^ (gm.dim > 2 ? z * 805459861u : 0u);
    } else {
        idx = x + y * gm.mul1[l] + z * gm.mul2[l];
    }
    // index % hashmap_size (gridencoder.cu:83).  Capped levels have a power-of-two size (2^log2_hashmap_size): one AND;
    // uncapped levels hold the whole dense grid, so the generic modulo is almost never taken.
    const uint32_t hm = gm.hmask[l];
    if (hm) return idx & hm;
    const uint32_t hs = gm.hsize[l];
    if (idx >= hs) idx %= hs;
    return idx;
}

// 3-D, C=2 interpolation of one level for a point in [0,1]^3.  Out-of-range input => zeros.
__device__ __forceinline__ float2 grid_lookup3(const GridMeta &gm, const float2 *__restrict__ table, int l, float u,
                                               float v, float w) {
    if (u < 0.f || u > 1.f || v < 0.f || v > 1.f || w < 0.f || w > 1.f) return make_float2(0.f, 0.f);
    const float s = gm.scale[l];
    float px = __fadd_rn(__fmul_rn(u, s), gm.align_off), py = __fadd_rn(__fmul_rn(v, s), gm.align_off),
          pz = __fadd_rn(__fmul_rn(w, s), gm.align_off);
    const float fx0 = floorf(px), fy0 = floorf(py), fz0 = floorf(pz);
    const uint32_t gx = (uint32_t)fx0, gy = (uint32_t)fy0, gz = (uint32_t)fz0;
    px -= fx0; py -= fy0; pz -= fz0;
    if (gm.interp == 1) {
        px = px * px * (3.0f - 2.0f * px);
        py = py * py * (3.0f - 2.0f * py);
        pz = pz * pz * (3.0f - 2.0f * pz);
    }
    const float2 *tb = table + gm.offset[l];
    float2 c[8];
    if (!gm.hashed[l]) {
        // tiled level: the 8 corner slots differ by fixed strides -- one base index, adds, and a mask (or the rare modulo)
        const uint32_t m1 = gm.mul1[l], m2 = gm.mul2[l], hm = gm.hmask[l], hs = gm.hsize[l];
        const uint32_t base = gx + gy * m1 + gz * m2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t idx = base + (i & 1) + ((i & 2) ? m1 : 0u) + ((i & 4) ? m2 : 0u);
            if (hm) idx &= hm;
            else if (idx >= hs) idx %= hs;
            c[i] = __ldg(tb + idx);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i)
            c[i] = __ldg(tb + grid_slot(gm, l, gx + (i & 1), gy + ((i >> 1) & 1), gz + ((i >> 2) & 1)));
    }
    // same factor order as the reference: w = 1; w *= (x term); w *= (y term); w *= (z term)
    const float wx[2] = {1.0f - px, px}, wy[2] = {1.0f - py, py}, wz[2] = {1.0f - pz, pz};
    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float wgt = wx[i & 1] * wy[(i >> 1) & 1] * wz[(i >> 2) & 1];
        acc.x += wgt * c[i].x;
        acc.y += wgt * c[i].y;
    }
    return acc;
}

// ---- sector-packed corner layout ("quads") ------------------------------------------------------------------------
// For tiled grids the corner slots of a cell are base + {0, 1, m1, m1+1} (+ m2 for the far z plane), so the table is
// re-laid out at pack time as 32-byte blocks  Q[i] = { T[i], T[i+1], T[i+m1], T[i+m1+1] }  (indices mod the level size):
// one 32-byte sector per (cell, z-plane) instead of four scattered 8-byte entries.  The gather is bound by the number of
// outstanding L1 misses x L2 latency; this cuts sectors per (sample, level) from ~4-8 to 2 and LDG instructions from 8 to 4.
// Costs 4x table memory (2 x 28.8 MB for the May head: more than the H100's 50 MB L2, yet still faster there than the
// reference layout, DESIGN.md section 4).  Values and arithmetic are
// unchanged, so results are bit-identical to the unpacked path.
__device__ __forceinline__ uint32_t grid_mod(const GridMeta &gm, int l, uint32_t idx) {
    const uint32_t hm = gm.hmask[l];
    if (hm) return idx & hm;
    const uint32_t hs = gm.hsize[l];
    return idx >= hs ? idx % hs : idx;
}

// one 32-byte read-only global load as two 16-byte loads of the same sector (Hopper has no 256-bit load); p must be 32-byte aligned
__device__ __forceinline__ void ldg256(const uint4 *p, uint4 &lo, uint4 &hi) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo.x), "=r"(lo.y), "=r"(lo.z), "=r"(lo.w) : "l"(p));
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(hi.x), "=r"(hi.y), "=r"(hi.z), "=r"(hi.w) : "l"(p + 1));
}
// same, streaming past L1 (no line allocated): the fp16 oct gathers of the 2-CTA kernel, which leaves L1 only ~28 KB
__device__ __forceinline__ void ldg256_na(const uint4 *p, uint4 &lo, uint4 &hi) {
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo.x), "=r"(lo.y), "=r"(lo.z), "=r"(lo.w) : "l"(p));
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(hi.x), "=r"(hi.y), "=r"(hi.z), "=r"(hi.w) : "l"(p + 1));
}
__device__ __forceinline__ float2 grid_lookup3q(const GridMeta &gm, const float4 *__restrict__ quads, int l, float u, float v, float w) {
    if (u < 0.f || u > 1.f || v < 0.f || v > 1.f || w < 0.f || w > 1.f) return make_float2(0.f, 0.f);
    const float s = gm.scale[l];
    float px = __fadd_rn(__fmul_rn(u, s), gm.align_off), py = __fadd_rn(__fmul_rn(v, s), gm.align_off),
          pz = __fadd_rn(__fmul_rn(w, s), gm.align_off);
    const float fx0 = floorf(px), fy0 = floorf(py), fz0 = floorf(pz);
    const uint32_t gx = (uint32_t)fx0, gy = (uint32_t)fy0, gz = (uint32_t)fz0;
    px -= fx0; py -= fy0; pz -= fz0;
    if (gm.interp == 1) {
        px = px * px * (3.0f - 2.0f * px);
        py = py * py * (3.0f - 2.0f * py);
        pz = pz * pz * (3.0f - 2.0f * pz);
    }
    const uint32_t m2 = gm.mul2[l];
    const uint32_t base = gx + gy * gm.mul1[l] + gz * m2;
    const float4 *qb = quads + 2 * (size_t)gm.offset[l];
    // (levels whose z stride was dropped -- m2 == 0, get_grid_index quirk H5 -- read the same block twice: an L1 hit; a
    //  branch to skip it measured slower)
    const uint32_t q0 = grid_mod(gm, l, base), q1 = grid_mod(gm, l, base + m2);
    uint4 ua0, ua1, ub0, ub1;
    ldg256(reinterpret_cast<const uint4 *>(qb + 2 * q0), ua0, ua1);
    ldg256(reinterpret_cast<const uint4 *>(qb + 2 * q1), ub0, ub1);
    const float4 a0 = *reinterpret_cast<float4 *>(&ua0), a1 = *reinterpret_cast<float4 *>(&ua1),
                 b0 = *reinterpret_cast<float4 *>(&ub0), b1 = *reinterpret_cast<float4 *>(&ub1);
    // same corner order and factor order as grid_lookup3: i = dx + 2 dy + 4 dz,  w = (x term) * (y term) * (z term)
    const float wx0 = 1.0f - px, wy0 = 1.0f - py, wz0 = 1.0f - pz;
    float2 acc = make_float2(0.f, 0.f);
    float wgt;
    wgt = wx0 * wy0 * wz0; acc.x += wgt * a0.x; acc.y += wgt * a0.y;
    wgt = px * wy0 * wz0;  acc.x += wgt * a0.z; acc.y += wgt * a0.w;
    wgt = wx0 * py * wz0;  acc.x += wgt * a1.x; acc.y += wgt * a1.y;
    wgt = px * py * wz0;   acc.x += wgt * a1.z; acc.y += wgt * a1.w;
    wgt = wx0 * wy0 * pz;  acc.x += wgt * b0.x; acc.y += wgt * b0.y;
    wgt = px * wy0 * pz;   acc.x += wgt * b0.z; acc.y += wgt * b0.w;
    wgt = wx0 * py * pz;   acc.x += wgt * b1.x; acc.y += wgt * b1.y;
    wgt = px * py * pz;    acc.x += wgt * b1.z; acc.y += wgt * b1.w;
    return acc;
}

// ---- fp16 "oct" layout (fp16 precision mode only) ------------------------------------------------------------------
// All eight corners of a cell, both features, as fp16: 8 x half2 = 32 bytes = ONE sector per (sample, level):
//   O[i] = { T[i], T[i+1], T[i+m1], T[i+m1+1], T[i+m2], T[i+m2+1], T[i+m2+m1], T[i+m2+m1+1] }   (indices mod the level size)
// Table values are rounded to fp16 -- exactly what the reference does under autocast (gridencoder/grid.py:43-44: the
// embeddings are cast to half) -- and interpolated in fp32.  Used together with fp16 MMA operands, never in the
// fp32 / bf16x3 modes.  Reader: lookup8o (head_tc_kernel.cu); writer: k_pack_octs (ops_kernels.cu).
__device__ __forceinline__ float2 grid_lookup2(const GridMeta &gm, const float2 *__restrict__ table, int l, float u,
                                               float v) {
    if (u < 0.f || u > 1.f || v < 0.f || v > 1.f) return make_float2(0.f, 0.f);
    const float s = gm.scale[l];
    float px = __fadd_rn(__fmul_rn(u, s), gm.align_off), py = __fadd_rn(__fmul_rn(v, s), gm.align_off);
    const float fx0 = floorf(px), fy0 = floorf(py);
    const uint32_t gx = (uint32_t)fx0, gy = (uint32_t)fy0;
    px -= fx0; py -= fy0;
    if (gm.interp == 1) {
        px = px * px * (3.0f - 2.0f * px);
        py = py * py * (3.0f - 2.0f * py);
    }
    const float2 *tb = table + gm.offset[l];
    float2 c[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) c[i] = __ldg(tb + grid_slot(gm, l, gx + (i & 1), gy + ((i >> 1) & 1), 0u));
    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float wgt = (i & 1) ? px : 1.0f - px;
        wgt *= (i & 2) ? py : 1.0f - py;
        acc.x += wgt * c[i].x;
        acc.y += wgt * c[i].y;
    }
    return acc;
}

// degree-4 real spherical harmonics (shencoder.cu:43-68)
__device__ __forceinline__ void sh4(float x, float y, float z, float *o) {
    const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

}  // namespace gfpp
