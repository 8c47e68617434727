// head_common.cuh -- ray-slot state and helpers shared by the two fused head kernels
// (head_kernel.cu: fp32 FFMA MLP; head_tc_kernel.cu: wgmma tensor-core MLP).
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"
#include "head_kernel.cuh"

namespace gfpp {
namespace headc {

namespace cg = cooperative_groups;

// add `val` to base[key] once per distinct key in the warp's active lanes
__device__ __forceinline__ void warp_agg_add(int *base, int key, int val) {
    const unsigned act = __activemask();
    const unsigned grp = __match_any_sync(act, key);
    const int sum = __reduce_add_sync(grp, val);
    if ((int)(__ffs(grp) - 1) == (int)(threadIdx.x & 31)) atomicAdd(base + key, sum);
}

struct Slot {
    RayGeom g;
    float t, near, far, ws, depth, r, gch, b;
    float T;       // transmittance as composite_rays_train carries it (training termination only; see composite_and_advance)
    float far_m;   // marching bound: min(far, exit of the padded occupied box) -- nothing is occupied beyond it
    float px, py, pz, dt;  // pending sample
    int gid, frame, nsamp, cap;
    bool active;
};

// What k_ray_setup leaves for the persistent kernel: a ray that reaches a first sample, ready to run.  One 64-byte record =
// two 256-bit loads on adoption instead of hit-id -> pose -> get_rays/near_far/box arithmetic between two CTA barriers.
struct alignas(32) HitRecord {
    int gid;
    float t, px, py, pz, dt;      // first sample (t already advanced past it)
    float near, far, far_m;
    float ox, oy, oz, dx, dy, dz;
    int pad;
};
static_assert(sizeof(HitRecord) == 64, "HitRecord is four 16-byte words");

__device__ __forceinline__ void load_ray(const HeadArgs &a, int frame, int ray, RayGeom &g) {
    if (a.rays_o) {
        const size_t o = ((size_t)frame * a.n_rays + ray) * 3;
        ray_geom_init(g, a.rays_o[o], a.rays_o[o + 1], a.rays_o[o + 2], a.rays_d[o], a.rays_d[o + 1], a.rays_d[o + 2]);
    } else {
        // get_rays (modules/radnerfs/utils.py:302-360): pixel centre, normalise, rotate by c2w[:3,:3]
        const float *P = a.poses + (size_t)frame * 16;
        const int row = ray / a.img_w, col = ray - row * a.img_w;
        const float xs = __fdiv_rn(__fsub_rn((float)col + 0.5f, a.cx), a.fx);
        const float ys = __fdiv_rn(__fsub_rn((float)row + 0.5f, a.cy), a.fy);
        const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(xs, xs), __fmul_rn(ys, ys)), 1.0f));
        const float dxc = __fdiv_rn(xs, nrm), dyc = __fdiv_rn(ys, nrm), dzc = __fdiv_rn(1.0f, nrm);
        float d[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            d[k] = __fadd_rn(__fadd_rn(__fmul_rn(dxc, P[4 * k]), __fmul_rn(dyc, P[4 * k + 1])), __fmul_rn(dzc, P[4 * k + 2]));
        ray_geom_init(g, P[3], P[7], P[11], d[0], d[1], d[2]);
    }
}

// conservative: can the segment [near, far] of the ray touch the (one-cell padded) box of occupied voxels?
// On return `far_m` is the parameter beyond which the ray cannot meet an occupied voxel (<= far): the marcher may stop
// there, which removes the long ALU-only walks of rays that have left the object.
__device__ __forceinline__ bool may_hit_occupied(bool have_box, const float (&occ_lo)[3], const float (&occ_hi)[3],
                                                 const RayGeom &g, float near, float far, float &far_m) {
    far_m = far;
    if (!have_box) return true;
    float t0 = near, t1 = far;
    const float o[3] = {g.ox, g.oy, g.oz}, rd[3] = {g.rdx, g.rdy, g.rdz}, d[3] = {g.dx, g.dy, g.dz};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (d[k] == 0.f) {
            if (o[k] < occ_lo[k] || o[k] > occ_hi[k]) return false;
            continue;
        }
        float ta = (occ_lo[k] - o[k]) * rd[k], tb = (occ_hi[k] - o[k]) * rd[k];
        if (ta > tb) { const float s = ta; ta = tb; tb = s; }
        t0 = fmaxf(t0, ta);
        t1 = fminf(t1, tb);
    }
    if (t0 <= t1) far_m = fminf(far, t1);
    return t0 <= t1;
}

__device__ __forceinline__ void finalize_ray(const HeadArgs &a, const Slot &s, bool normalise_depth) {
    const size_t g = (size_t)s.gid;
    a.image[3 * g] = s.r;
    a.image[3 * g + 1] = s.gch;
    a.image[3 * g + 2] = s.b;
    a.wsum[g] = s.ws;
    // renderer.py:394: depth = clamp(depth - nears, min=0) / (fars - nears)
    a.depth[g] = normalise_depth ? __fdiv_rn(fmaxf(__fsub_rn(s.depth, s.near), 0.f), __fsub_rn(s.far, s.near)) : s.depth;
}



// padded world-space box of the occupied voxels (cascade 0) from the device-side cell bounds; also installs the cell
// bounds into `mc`.  Rays whose [near, far] segment misses the box have no sample.
__device__ __forceinline__ bool setup_occupancy(const HeadArgs &a, MarchConst &mc, float (&occ_lo)[3], float (&occ_hi)[3]) {
    bool have_box = false;
    if (a.occ_bounds) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { mc.bb_lo[k] = a.occ_bounds[k]; mc.bb_hi[k] = a.occ_bounds[3 + k]; }
        if (a.use_occ_box) {
            have_box = true;
            const float mb = fminf(1.0f, mc.bound);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (mc.bb_hi[k] < mc.bb_lo[k]) { occ_lo[k] = 1e30f; occ_hi[k] = -1e30f; }  // nothing occupied
                else {
                    occ_lo[k] = ((float)(mc.bb_lo[k] - 1) * mc.rH * 2.0f - 1.0f) * mb;
                    occ_hi[k] = ((float)(mc.bb_hi[k] + 2) * mc.rH * 2.0f - 1.0f) * mb;
                }
            }
        }
    }
    return have_box;
}

constexpr int kFetchTries = 4;   // rays a thread may try per refill iteration (most candidates are cheap misses)
constexpr int kRefillIters = 2;

// Refill dead slots from the global work cursor, then publish the batch (valid flags, frame ids, sample positions).
// Returns the number of valid rows, or -1 when the CTA is out of work.  All threads of the CTA must call it.
template <class SmemT>
__device__ __forceinline__ int refill_and_publish(const HeadArgs &a, SmemT &s, Slot &sl, const MarchConst &mc, bool have_box,
                                                  const float (&occ_lo)[3], const float (&occ_hi)[3], int total, int tid) {
    constexpr int TM = HEAD_TM;
    for (int it = 0; it < kRefillIters; ++it) {
        if (tid == 0 && s.next >= s.end && !s.done) {
            const int base = atomicAdd(a.cursor, TM);
            if (base >= total) { s.done = 1; }
            else { s.next = base; s.end = min(base + TM, total); }
        }
        __syncthreads();
        if (tid < TM && !sl.active) {
            for (int attempt = 0; attempt < kFetchTries && !sl.active && s.next < s.end; ++attempt) {
                const int w = atomicAdd(&s.next, 1);
                if (w >= s.end) break;
                int gid;
                HitRecord hr;
                if (a.pass == 2) {
                    gid = a.survivors[w];
                    sl.gid = gid;
                    sl.frame = gid / a.n_rays;
                    load_ray(a, sl.frame, gid - sl.frame * a.n_rays, sl.g);
                    near_far(sl.g, a.aabb, a.min_near, sl.near, sl.far);
                } else {
                    uint4 *q = reinterpret_cast<uint4 *>(&hr);
                    ldg256(a.hits + 4 * (size_t)w, q[0], q[1]);
                    ldg256(a.hits + 4 * (size_t)w + 2, q[2], q[3]);
                    gid = hr.gid;
                    sl.gid = gid;
                    sl.frame = gid / a.n_rays;
                }
                bool live;
                if (a.pass == 1) {
                    // k_ray_setup already set this ray up and marched it to its first sample: adopt the record
                    ray_geom_init(sl.g, hr.ox, hr.oy, hr.oz, hr.dx, hr.dy, hr.dz);
                    sl.near = hr.near; sl.far = hr.far; sl.far_m = hr.far_m;
                    sl.t = hr.t; sl.px = hr.px; sl.py = hr.py; sl.pz = hr.pz; sl.dt = hr.dt;
                    sl.ws = 0.f; sl.depth = 0.f; sl.r = sl.gch = sl.b = 0.f; sl.T = 1.f;
                    sl.nsamp = 0; sl.cap = a.max_steps;
                    live = true;
                } else {
                    const size_t g = (size_t)gid;
                    sl.t = a.rays_t[g]; sl.ws = a.wsum[g]; sl.depth = a.depth[g];
                    sl.r = a.image[3 * g]; sl.gch = a.image[3 * g + 1]; sl.b = a.image[3 * g + 2];
                    sl.nsamp = a.max_steps; sl.cap = a.B_total[sl.frame];
                    (void)may_hit_occupied(have_box, occ_lo, occ_hi, sl.g, sl.near, sl.far, sl.far_m);
                    live = sl.nsamp < sl.cap && march_next(mc, sl.g, sl.far_m, sl.t, sl.px, sl.py, sl.pz, sl.dt);
                    if (!live) finalize_ray(a, sl, true);
                }
                sl.active = live;
            }
        }
        // another iteration only pays off when slots are still empty AND the local chunk ran dry while work remains
        const int want_more = __syncthreads_or(tid < TM && !sl.active && s.next >= s.end && !s.done);
        if (!want_more) break;
    }
    if (tid < TM) {
        s.valid[tid] = sl.active ? 1 : 0;
        s.frame[tid] = sl.frame;
        s.sx[tid] = sl.px; s.sy[tid] = sl.py; s.sz[tid] = sl.pz;
    }
    const int n_valid = __syncthreads_count(tid < TM && sl.active);
    if (n_valid == 0) {
        const bool out_of_work = s.done && s.next >= s.end;
        __syncthreads();  // thread 0 must not start the next refill (which rewrites next/end/done) before everyone has read them
        return out_of_work ? -1 : 0;
    }
    return n_valid;
}

// Front-to-back compositing of the batch's sample in the owner thread (raymarching.cu:978-1006), termination test,
// then march to the ray's next sample (or retire the ray).
// TRAIN: the termination of composite_rays_train (raymarching.cu:647-667) instead, for the frozen head of the torso training
// step (gfpp_frozen_head, pass 1 only): T is the running product of (1 - alpha) and the ray stops after the sample that takes
// it below T_thresh.  Inference uses T = 1 - weights_sum before the sample and stops one sample later.
template <bool TRAIN = false, class SmemT>
__device__ __forceinline__ void composite_and_advance(const HeadArgs &a, SmemT &s, Slot &sl, const MarchConst &mc, int tid) {
    constexpr int TM = HEAD_TM;
    if (tid < TM && sl.active) {
        const float sigma = s.sig[tid];
        const float alpha = 1.0f - expf(-sigma * sl.dt);
        const float T = TRAIN ? sl.T : 1.0f - sl.ws;
        const float w = alpha * T;
        if (TRAIN) sl.T = T * (1.0f - alpha);
        sl.ws += w;
        sl.depth += w * sl.t;  // sl.t is already the post-sample t (deltas[1])
        sl.r += w * s.rgb[tid];
        sl.gch += w * s.rgb[TM + tid];
        sl.b += w * s.rgb[2 * TM + tid];
        sl.nsamp += 1;
        if (a.valid_samples) warp_agg_add(a.valid_samples, sl.frame, 1);
        int D = 0;  // death index (1-based sample position), 0 = still alive
        bool suspend = false;
        if ((TRAIN ? sl.T : T) < a.T_thresh) D = sl.nsamp;
        else if (sl.nsamp >= sl.cap) suspend = true;
        else if (!march_next(mc, sl.g, sl.far_m, sl.t, sl.px, sl.py, sl.pz, sl.dt)) D = sl.nsamp + 1;
        if (D) {
            finalize_ray(a, sl, true);
            if (a.pass == 1) warp_agg_add(a.hist, sl.frame * (a.max_steps + 2) + D, 1);
            sl.active = false;
        } else if (suspend) {
            if (a.pass == 1) {
                finalize_ray(a, sl, false);  // raw depth: pass 2 keeps accumulating
                a.rays_t[sl.gid] = sl.t;
                cg::coalesced_group grp = cg::coalesced_threads();
                int base = 0;
                if (grp.thread_rank() == 0) base = atomicAdd(a.n_survivors, (int)grp.size());
                base = grp.shfl(base, 0);
                a.survivors[base + grp.thread_rank()] = sl.gid;
            } else {
                finalize_ray(a, sl, true);
            }
            sl.active = false;
        }
    }
}

// copy the coarse occupancy words into shared memory and point the marcher at them
template <class SmemT>
__device__ __forceinline__ void install_coarse(const HeadArgs &a, SmemT &s, MarchConst &mc, int tid, int nthreads) {
    if (a.coarse_bits && a.coarse_words <= HEAD_COARSE_WORDS) {
        for (int i = tid; i < a.coarse_words; i += nthreads) s.coarse[i] = a.coarse_bits[i];
        mc.coarse = s.coarse;
    } else {
        mc.coarse = a.coarse_bits;   // too large for the smem slot (cascade > 2): read through L1/L2
    }
}

}  // namespace headc
}  // namespace gfpp
