// head_v2_kernel.cu -- fused persistent head renderer, second generation (wgmma + bulk-copy weight stream).
//
// Replaces the reference's host-driven round loop (modules/radnerfs/renderer.py:340-384: march_rays -> GridEncoder ->
// ambient MLP -> GridEncoder -> sigma MLP -> SHEncoder -> color MLP -> composite_rays, ~40 launches per round) like
// head_tc_kernel.cu does, but organised around ROW OWNERSHIP instead of CTA-wide phases:
//
//   * one CTA per SM; NSLOT "slots" of 128 samples, each one warpgroup whose thread r owns row r: the ray, the gather of the
//     row's grid levels into its 16-bit operand row, and the row's scalars in registers;
//   * the warpgroup runs its own layers with wgmma, rows 0-63 then 64-127 (fp32 accumulators in registers), each half's
//     epilogue straight from the accumulator fragment (the halves touch disjoint operand rows); while one slot's MMAs run,
//     the other slots do their gathers and ray work;
//   * the weight stream is SHARED: the loader warp copies each tile once (NSTAGE-deep ring) for all slots; a stage is refilled
//     once every owner warp has arrived on `w_free`;
//   * the 3-wide outputs and the sigma logit are N=16 MMAs against small RESIDENT tiles, handed to the row owners through a
//     small buffer at the head of the slot's second operand tile (the sigma logit through a per-row buffer of its own);
//   * the CTA is whole warpgroups: NSLOT owner warpgroups and one producer warpgroup, whose registers (setmaxnreg) go to
//     the owners;
//   * fp16: the position-grid features of a row's NEXT sample are looked up by the slot's GATHER WARP (producer warp 1 + s) while
//     the slot runs its layers, and handed over through a per-row staging slot, so the owners never wait on those loads.
//
// Precision modes: FP16_X1 (the reference's autocast arithmetic) with 3 slots, and FP16_ROBUST with 2 slots: fp16 hi/lo
// split (3 MMAs per k-step, ~22 mantissa bits) on the ambient net and a 16-bit fixed-point position table (gather8.cuh) --
// the two roundings the field amplifies (tools/error_budget.py) -- everything else as FP16_X1.
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "gather8.cuh"
#include "head_common.cuh"
#include "head_kernel.cuh"
#include "launch.cuh"
#include "tc.cuh"

namespace gfpp {

using namespace tc;
using namespace headc;

namespace {

constexpr int TM = HEAD_TM;          // rows per slot
// fp16: the first position level the gather warps look up; the owners look up levels [0, GATHER_L0) themselves, into the same
// staging row.  0: the gather warps take all 16 levels; 8: the owners keep levels 0-7.  On an H100 80GB HBM3 (700 W) with the
// bench's tables one warp per slot does not finish 16 levels in the shadow of the slot's layers (the "wait for staged position
// features" stamp: 11 k cycles per batch at 0, 1.3 k at 8)
constexpr int GATHER_L0 = 8;
constexpr int GATHER_N = 2;          // levels per lookup call of a gather warp: 2 x 32-byte loads in flight per lane (56 registers, no spills)
static_assert(GATHER_L0 == 0 || GATHER_L0 == 8, "the owners gather whole 8-level halves");
static_assert(GATHER_N % 2 == 0 && 8 % GATHER_N == 0, "a lookup call of a gather warp stores whole 8-byte pairs of levels");

template <bool ROBUST>
struct Cfg {
    static constexpr int NSLOT = ROBUST ? 2 : 3;
    static constexpr int NSTAGE = 4;   // >= 4: a robust ambient layer waits for four tiles at once
    static constexpr int NTILE = ROBUST ? V2_NTILE_ROBUST : V2_NTILE_X1;
    static constexpr int NWORK = 4 * NSLOT;                 // row-owner warps
    static constexpr int NT = 128 * (NSLOT + 1);            // + one producer warpgroup: its warp 0 is the loader
    // fp16: producer warps 1..NSLOT are the slots' gather warps and the owners read the position features from the staging rows;
    // the robust mode has no shared memory left for staging and gathers in the owners
    static constexpr bool STAGED = !ROBUST;
    static constexpr int OWN_LV = STAGED ? GATHER_L0 : 16;  // position levels the owners look up themselves
    // register split (setmaxnreg): the owner warpgroups grow to OWNER_REGS, the producer warpgroup shrinks to PRODUCER_REGS.
    // The launch allocates 65536 / NT per thread (128 | 168); the owners' increase is served by the producer's decrease.
    static constexpr int OWNER_REGS = ROBUST ? 232 : 152, PRODUCER_REGS = ROBUST ? 40 : 56;
    static constexpr int LAUNCH_REGS = (65536 / NT) & ~7;
    static_assert(NSLOT * 128 * OWNER_REGS + 128 * PRODUCER_REGS <= 65536, "register split exceeds the register file");
    static_assert(NSLOT * 128 * (OWNER_REGS - LAUNCH_REGS) <= 128 * (LAUNCH_REGS - PRODUCER_REGS), "owners grow by more than the producer frees");
    static_assert(OWNER_REGS % 8 == 0 && PRODUCER_REGS % 8 == 0 && PRODUCER_REGS >= 24 && OWNER_REGS <= 256, "setmaxnreg operand");
    static constexpr int SLOT_BYTES = (ROBUST ? 4 : 2) * V2_TILE_BYTES + 4096;   // h0 h1 [l0 l1] sh
    static constexpr int OFF_W = NSLOT * SLOT_BYTES;
    static constexpr int OFF_RES = OFF_W + NSTAGE * V2_TILE_BYTES;
    static constexpr int OFF_MISC = OFF_RES + V2_RES_BYTES;
};

struct Misc {
    float cbias[128];                    // color L0 bias (individual code folded)
    uint32_t coarse[HEAD_COARSE_WORDS];
    uint4 lvl[2][2 * GFPP_MAX_LEVELS];
    MarchConst mc;
    float occ_lo[3], occ_hi[3];
    bool have_box;
    unsigned long long w_full[4], w_free[4], res_full, batch_bar;
    // fp16, per slot, one phase per batch: the owners have posted their rows' next coordinates (TM arrivals) | the gather warp
    // has staged their features (32 arrivals); `pos_quit`: the owners' last request, the gather warp leaves
    unsigned long long pos_req[3], pos_done[3];
    volatile int pos_quit[3];
    volatile int stop;
    volatile int flag[2][16];            // per batch parity, per owner warp: "I have live rows"
};

// the sigma logits of a slot's rows, from the sigma row's MMA (issued with color L0) to the row owners (TM floats per slot): the
// robust mode keeps them at the head of the slot's residual tile l (idle from ambient out to the next batch's operand rows), fp16
// behind Misc
template <bool ROBUST>
constexpr size_t slogit_bytes() { return ROBUST ? 0 : (size_t)Cfg<ROBUST>::NSLOT * TM * sizeof(float); }
// fp16: the gather warps' staging rows behind the sigma logits, [NSLOT][TM] x 64 bytes: 16 levels as packed fp16 pairs (level j
// in 32-bit word j) or, from the owner's post to the gather warp's reply, the row's next grid coordinates in chunk 0
template <bool ROBUST>
constexpr size_t stage_bytes() { return Cfg<ROBUST>::STAGED ? (size_t)Cfg<ROBUST>::NSLOT * TM * 64 : 0; }
template <bool ROBUST>
constexpr size_t smem_bytes() { return (size_t)Cfg<ROBUST>::OFF_MISC + sizeof(Misc) + slogit_bytes<ROBUST>() + stage_bytes<ROBUST>() + 1024; }
static_assert(smem_bytes<false>() <= 227 * 1024 && smem_bytes<true>() <= 227 * 1024, "v2 shared memory budget");

// Epilogue of one M = 64 half (rows 64*half ..) of a 128-wide layer from the accumulator fragment: (+bias) -> (ReLU) ->
// operand tiles h0|h1 (cols 0-63 | 64-127) and, when LO, the residual images l0|l1.  BIAS: shared-memory vector (color L0).
template <bool RELU, bool BIAS, bool LO>
__device__ __forceinline__ void epilogue_half(const float (&d)[64], unsigned char *h, unsigned char *l, int half, int lane, int wwarp,
                                              const float *bias) {
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int row = 64 * half + frag_row(i, lane, wwarp), col = frag_col(i, lane);
        float x0 = d[i], x1 = d[i + 1];
        if (BIAS) { x0 += bias[col]; x1 += bias[col + 1]; }
        if (RELU) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        store_pair<false, LO>(h + (col >> 6) * V2_TILE_BYTES, l + (LO ? (col >> 6) * V2_TILE_BYTES : 0), row, col & 63, x0, x1);
    }
}

// per-thread register budget of the executing warpgroup (all four warps, converged)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ float2 unpack_h2(uint32_t h) { return __half22float2(*reinterpret_cast<const __half2 *>(&h)); }

// 16-byte chunk c of staging row `row`: chunks rotate with row / 2, so that eight consecutive rows' 16-byte accesses (the owners'
// and the gather warp's) fall on distinct banks
__device__ __forceinline__ uint32_t stage_off(int row, int c) { return (uint32_t)row * 64u + (uint32_t)((c ^ (row >> 1)) & 3) * 16u; }

// N = 16 group over K = 128: operand tiles a | a + one tile against the two 2 KB halves of a resident tile at w
__device__ __forceinline__ void mma16(float (&d)[8], uint32_t a, uint32_t w, uint32_t acc_first) {
    wgmma_sw<16, false>(d, a, w, 4, acc_first);
    wgmma_sw<16, false>(d, a + V2_TILE_BYTES, w + 2048, 4, 1u);
}

// Columns c0 .. c0+NC-1 of an N = 16 accumulator fragment -> out[c][row] (rows of this half), read back by the row owners
template <int NC>
__device__ __forceinline__ void put_cols(const float (&d)[8], float *out, int c0, int half, int lane, int wwarp) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int col = frag_col(i, lane) - c0;
        if (col >= 0 && col < NC) out[col * TM + 64 * half + frag_row(i, lane, wwarp)] = d[i];
    }
}

// warp-level feed of hit-list / survivor-list indices: a chunk of 32 consecutive entries is claimed with ONE global atomic and
// handed out to the lanes that need a ray (uniform across the warp)
struct WarpFeed { int next, end; bool dry; };

}  // namespace

// the conditioning vectors of the clip as fp16 operand images: hi = rn16(x), lo = rn16(x - hi)  (64 values = 128 bytes per frame)
__global__ void k_cond_images(const float *__restrict__ cond /*[F,64]*/, int n, __half *__restrict__ hi, __half *__restrict__ lo) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = cond[i];
    const __half h = __float2half_rn(x);
    hi[i] = h;
    lo[i] = __float2half_rn(x - __half2float(h));
}

template <bool ROBUST, bool PROFILE>
__global__ void __launch_bounds__(Cfg<ROBUST>::NT, 1) k_head_v2(const __grid_constant__ HeadArgs a, const __grid_constant__ HeadV2Args t) {
    using C = Cfg<ROBUST>;
    constexpr int NSTAGE = C::NSTAGE, NTILE = C::NTILE, NWORK = C::NWORK;
    extern __shared__ __align__(1024) unsigned char smem_raw_[];
    unsigned char *sm = smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u);
    Misc &ms = *reinterpret_cast<Misc *>(sm + C::OFF_MISC);
    unsigned char *wring = sm + C::OFF_W, *res = sm + C::OFF_RES;
    unsigned char *stage = sm + C::OFF_MISC + sizeof(Misc) + slogit_bytes<ROBUST>();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    // ---------------- one-time setup ----------------
    const bool coarse_in_smem = a.coarse_bits && a.coarse_words <= HEAD_COARSE_WORDS;
    if (coarse_in_smem)
        for (int i = tid; i < a.coarse_words; i += C::NT) ms.coarse[i] = a.coarse_bits[i];
    if (tid == 0) {
        // marching constants and the occupied box in shared memory, not in ~25 registers of every owner thread
        ms.mc = a.mc;
        for (int k = 0; k < 3; ++k) { ms.occ_lo[k] = 0.f; ms.occ_hi[k] = 0.f; }
        ms.have_box = setup_occupancy(a, ms.mc, ms.occ_lo, ms.occ_hi);
        ms.mc.coarse = coarse_in_smem ? ms.coarse : a.coarse_bits;
        for (int i = 0; i < 4; ++i) { mbar_init(&ms.w_full[i], 1); mbar_init(&ms.w_free[i], NWORK); }
        mbar_init(&ms.res_full, 1);
        mbar_init(&ms.batch_bar, NWORK);
        if (C::STAGED)
            for (int i = 0; i < C::NSLOT; ++i) { mbar_init(&ms.pos_req[i], TM); mbar_init(&ms.pos_done[i], 32); ms.pos_quit[i] = 0; }
        mbar_fence_init();
        ms.stop = 0;
    }
    if (tid < 128) ms.cbias[tid] = a.narrow[7 * 128 + tid];
    if (tid < 32) { ms.flag[0][tid & 15] = 0; ms.flag[1][tid & 15] = 0; }
    stage_level_meta(a.pos_gm, ROBUST ? t.pos_step : nullptr, ms.lvl[0], tid);
    stage_level_meta(a.amb_gm, nullptr, ms.lvl[1], tid);
    fence_async_smem();
    __syncthreads();
    const int total = (a.pass == 1) ? *a.n_hits : *a.n_survivors;

    if (warp < NWORK) {
        setmaxnreg_inc<C::OWNER_REGS>();
        // =====================================================================================================
        // ROW OWNER: thread `row` of slot `s`
        //
        // Software-pipelined over the sample sequence of its rays: `cu` is the sample being shaded in this batch, `sl` already
        // holds the NEXT one.  What happens to the ray after the current sample -- it dies because T < T_thresh (T uses the
        // weights BEFORE this sample, raymarching.cu:1000-1004), it reaches its sample cap, or marching runs off the volume --
        // does not depend on the sample's own sigma, so the march to the next sample, the adoption of a new ray and the gather
        // of the next sample's position features all run in the shadow of the current batch's MMAs.
        // =====================================================================================================
        const int s = warp >> 2, row = tid & (TM - 1), wwarp = warp & 3;
        unsigned char *h = sm + s * C::SLOT_BYTES, *l = h + 2 * V2_TILE_BYTES, *sht = h + (ROBUST ? 4 : 2) * V2_TILE_BYTES;
        // live columns of the N = 16 layers, [3][TM] floats at the head of tile h1: they only overlap operand rows 0-15 of h1,
        // which half 0 has consumed before they are written and which are rewritten only after the owners have read them
        float *outc = reinterpret_cast<float *>(h + V2_TILE_BYTES);
        float *slogit = ROBUST ? reinterpret_cast<float *>(l) : reinterpret_cast<float *>(sm + C::OFF_MISC + sizeof(Misc)) + s * TM;
        const uint32_t h_u = smem_u32(h), l_u = smem_u32(l), sh_u = smem_u32(sht), res_u = smem_u32(res), ring_u = smem_u32(wring);
        const MarchConst &mc = ms.mc;
        uint32_t wc = 0;            // streamed tiles consumed so far (the same sequence in every slot)
        const bool smooth_p = a.pos_gm.interp == 1, smooth_a = a.amb_gm.interp == 1;
        Slot sl;
        sl.active = false;
        sl.gid = 0; sl.frame = 0; sl.nsamp = 0; sl.cap = 0;
        sl.px = sl.py = sl.pz = 0.f; sl.dt = 0.f; sl.t = 0.f; sl.ws = 0.f; sl.depth = 0.f; sl.r = sl.gch = sl.b = 0.f;
        sl.near = sl.far = sl.far_m = 0.f;
        ray_geom_init(sl.g, 0.f, 0.f, 0.f, 1.f, 1.f, 1.f);
        WarpFeed wf{0, 0, false};
        uint32_t bpar = 0;
        bool newray = false;      // sl holds a freshly adopted ray whose SH operand row is not written yet
        // the sample being shaded: accumulators BEFORE it, its dt / post-sample t, and what happens to its ray afterwards
        struct { bool valid; int fate, D, gid, frame, nsamp; float dt, t_post, ws, depth, r, g, b, near, far; } cu;
        cu.valid = false; cu.fate = 0; cu.D = 0; cu.gid = 0; cu.frame = 0; cu.nsamp = 0;
        cu.dt = cu.t_post = cu.ws = cu.depth = cu.r = cu.g = cu.b = cu.near = cu.far = 0.f;
        // robust: position features of the current sample (packed fp16 pairs), looked up during the previous batch
        uint32_t feat[C::STAGED ? 1 : 16];
        unsigned char *stg = stage + s * TM * 64;   // fp16: this slot's staging rows
        uint32_t featl[ROBUST ? 16 : 1];

        // operand rows written by this warpgroup -> visible to its MMAs
#define ARRIVE_A()                                   \
    do {                                             \
        fence_async_smem();                          \
        wg_sync(1 + s);                              \
    } while (0)
        // wait for streamed tile wc + j, return its shared-memory address
        auto tile = [&](uint32_t j) -> uint32_t {
            const uint32_t i = wc + j, stage = i % NSTAGE;
            mbar_wait(&ms.w_full[stage], (i / NSTAGE) & 1u);
            return ring_u + stage * V2_TILE_BYTES;
        };
        // the n tiles just used are free for this warp (its MMAs have completed); a stage is refilled once every owner warp arrived
        auto release = [&](uint32_t n) {
            if (lane == 0)
                for (uint32_t j = 0; j < n; ++j) mbar_arrive(&ms.w_free[(wc + j) % NSTAGE]);
            __syncwarp();
            wc += n;
        };
        // one 128-wide layer against `ntile` streamed tiles: per M-half, `mma(d, half offset, w0, w1)` then `epi(d, half)`
        auto layer128 = [&](int ntile, auto &&mma, auto &&epi) {
            const uint32_t w0 = tile(0), w1 = ntile > 1 ? tile(1) : w0;
#pragma unroll 1
            for (int hf = 0; hf < 2; ++hf) {
                float d[64];
                wg_fence();
                mma(d, (uint32_t)hf * SW128_HALF, w0, w1);
                wg_commit();
                wg_wait<0>();
                acc_fence(d);
                epi(d, hf);
            }
            release((uint32_t)ntile);
        };
        // optional phase stamps (thread 0 = row 0 of slot 0 of every CTA): cycles between consecutive PH() points
        long long ph_last = clock64();
#define PH(i)                                                                              \
    if (PROFILE && a.phase_cycles && tid == 0) {                                                      \
        const long long now_ = clock64();                                                  \
        atomicAdd(a.phase_cycles + (i), (unsigned long long)(now_ - ph_last));             \
        ph_last = now_;                                                                    \
    }

        // refill dead lanes of `sl` from the warp's feed (all lanes of the warp, converged).  Pass 1 fills every dead lane within
        // two tries (each hit record is a live ray); in pass 2 a survivor already at its cap is finalised on adoption, so a warp
        // may go through many rounds before it holds a live ray, and every round given up is an empty batch
        auto refill = [&]() {
#pragma unroll 1
            for (int tries = 0; tries < 64; ++tries) {
                const unsigned need = __ballot_sync(0xffffffffu, !sl.active);
                if (!need) break;
                if (wf.next >= wf.end) {
                    if (wf.dry) break;
                    int base = 0;
                    if (lane == 0) base = atomicAdd(a.cursor, 32);
                    base = __shfl_sync(0xffffffffu, base, 0);
                    if (base >= total) { wf.dry = true; break; }
                    wf.next = base;
                    wf.end = min(base + 32, total);
                }
                const int rank = __popc(need & ((1u << lane) - 1u)), avail = wf.end - wf.next;
                const bool take = !sl.active && rank < avail;
                const int w = wf.next + rank;
                wf.next += min(__popc(need), avail);
                if (take) {
                    bool live;
                    if (a.pass == 1) {
                        // k_ray_setup already set this ray up and marched it to its first sample: adopt the 64-byte record
                        HitRecord hr;
                        uint4 *q = reinterpret_cast<uint4 *>(&hr);
                        ldg256(a.hits + 4 * (size_t)w, q[0], q[1]);
                        ldg256(a.hits + 4 * (size_t)w + 2, q[2], q[3]);
                        sl.gid = hr.gid;
                        sl.frame = hr.gid / a.n_rays;
                        ray_geom_init(sl.g, hr.ox, hr.oy, hr.oz, hr.dx, hr.dy, hr.dz);
                        sl.near = hr.near; sl.far = hr.far; sl.far_m = hr.far_m;
                        sl.t = hr.t; sl.px = hr.px; sl.py = hr.py; sl.pz = hr.pz; sl.dt = hr.dt;
                        sl.ws = 0.f; sl.depth = 0.f; sl.r = sl.gch = sl.b = 0.f;
                        sl.nsamp = 0; sl.cap = a.max_steps;
                        live = true;
                    } else {
                        const int gid = a.survivors[w];
                        sl.gid = gid;
                        sl.frame = gid / a.n_rays;
                        load_ray(a, sl.frame, gid - sl.frame * a.n_rays, sl.g);
                        near_far(sl.g, a.aabb, a.min_near, sl.near, sl.far);
                        const size_t g = (size_t)gid;
                        sl.t = a.rays_t[g]; sl.ws = a.wsum[g]; sl.depth = a.depth[g];
                        sl.r = a.image[3 * g]; sl.gch = a.image[3 * g + 1]; sl.b = a.image[3 * g + 2];
                        sl.nsamp = a.max_steps; sl.cap = a.B_total[sl.frame];
                        (void)may_hit_occupied(ms.have_box, ms.occ_lo, ms.occ_hi, sl.g, sl.near, sl.far, sl.far_m);
                        live = sl.nsamp < sl.cap && march_next(mc, sl.g, sl.far_m, sl.t, sl.px, sl.py, sl.pz, sl.dt);
                        if (!live) finalize_ray(a, sl, true);
                    }
                    sl.active = live;
                    newray = live;
                }
                __syncwarp();
            }
            // the records the warp will adopt next (64 B each, read once, from L2 or DRAM): pull them towards L1 a batch ahead
            if (a.pass == 1 && wf.next + lane < wf.end)
                asm volatile("prefetch.global.L1 [%0];" ::"l"(a.hits + 4 * (size_t)(wf.next + lane)));
        };
        // eight levels [8 * half, 8 * half + 8) of the position grid at the NEXT sample -> feat / featl
        auto prefetch_pos = [&](int half) {
            float f[16];
            if (sl.active) {
                const float inv2b = 2.0f * mc.bound;
                const float u = __fdiv_rn(__fadd_rn(sl.px, mc.bound), inv2b), vv = __fdiv_rn(__fadd_rn(sl.py, mc.bound), inv2b),
                            w = __fdiv_rn(__fadd_rn(sl.pz, mc.bound), inv2b);
                lookup8<ROBUST ? OCT_I16 : OCT_F16>(&ms.lvl[0][half * 16], a.pos_gm.align_off, smooth_p, a.pos_octs, u, vv, w, f);
            } else {
#pragma unroll
                for (int i = 0; i < 16; ++i) f[i] = 0.f;
            }
            if constexpr (C::STAGED) {   // the staging row's chunks of these levels: the gather warp only touches chunks [GATHER_L0 / 4, 4)
#pragma unroll
                for (int k = 0; k < 2; ++k)
                    *reinterpret_cast<uint4 *>(stg + stage_off(row, 2 * half + k)) =
                        make_uint4(pack2<false>(f[8 * k], f[8 * k + 1]), pack2<false>(f[8 * k + 2], f[8 * k + 3]),
                                   pack2<false>(f[8 * k + 4], f[8 * k + 5]), pack2<false>(f[8 * k + 6], f[8 * k + 7]));
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const uint32_t hi = pack2<false>(f[2 * i], f[2 * i + 1]);
                    feat[half * 8 + i] = hi;
                    if (ROBUST) {
                        const float2 b = unpack_h2(hi);
                        featl[half * 8 + i] = pack2<false>(f[2 * i] - b.x, f[2 * i + 1] - b.y);
                    }
                }
            }
        };
        // 16-byte chunk c (levels 4c .. 4c+3) of the current sample's position features
        auto pos_chunk = [&](int c) -> uint4 {
            if constexpr (C::STAGED) return *reinterpret_cast<const uint4 *>(stg + stage_off(row, c));
            else return make_uint4(feat[4 * c], feat[4 * c + 1], feat[4 * c + 2], feat[4 * c + 3]);
        };
        // fp16: the NEXT sample's grid coordinates -> the row's staging slot, a request to the slot's gather warp.  An inactive row
        // posts a point outside the grid, whose features are zeros
        auto post_pos = [&]() {
            float u = -1.f, vv = -1.f, w = -1.f;
            if (sl.active) {
                const float inv2b = 2.0f * mc.bound;
                u = __fdiv_rn(__fadd_rn(sl.px, mc.bound), inv2b);
                vv = __fdiv_rn(__fadd_rn(sl.py, mc.bound), inv2b);
                w = __fdiv_rn(__fadd_rn(sl.pz, mc.bound), inv2b);
            }
            *reinterpret_cast<float4 *>(stg + stage_off(row, GATHER_L0 / 4)) = make_float4(u, vv, w, 0.f);
            mbar_arrive(&ms.pos_req[s]);
        };
        // make `cu` the sample `sl` points at
        auto rotate = [&]() {
            cu.valid = sl.active;
            cu.dt = sl.dt; cu.t_post = sl.t;
            cu.ws = sl.ws; cu.depth = sl.depth; cu.r = sl.r; cu.g = sl.gch; cu.b = sl.b;
            cu.gid = sl.gid; cu.frame = sl.frame; cu.near = sl.near; cu.far = sl.far; cu.nsamp = sl.nsamp;
        };

        // ---------------- prologue: first rays, first samples, their position features ----------------
        refill();
        if (C::OWN_LV > 0) prefetch_pos(0);
        if (C::OWN_LV > 8) prefetch_pos(1);
        if (C::STAGED) post_pos();
        rotate();
        mbar_wait(&ms.res_full, 0);   // the resident N = 16 / SH weight tiles

        for (;;) {
            const bool valid = cu.valid;
            {   // batch accounting: this warp's "live rows" flag, then the split-phase batch barrier.  A warp whose feed is not dry
                // keeps the CTA going without live rows: the rays its next refill adopts must still get a batch
                const unsigned any = __ballot_sync(0xffffffffu, valid);
                if (lane == 0) {
                    ms.flag[bpar][warp] = (any || !wf.dry) ? 1 : 0;
                    mbar_arrive(&ms.batch_bar);
                }
            }
            if (C::STAGED) {   // the gather warp's reply to the request posted during the previous batch (or the prologue)
                mbar_wait(&ms.pos_done[s], bpar);
                PH(6)   // wait for staged position features
            }
            // ---------------- ambient-net input: h0 k[0,32) <- position features, k[32,64) | h1 k[0,32) <- conditioning ----------------
            if (newray && valid) {   // SH(dir) is constant along the ray: its K16 operand row is written once per ray (shencoder.cu:43-68)
                float shv[16];
                sh4(sl.g.dx, sl.g.dy, sl.g.dz, shv);
                store_chunk<false, false>(sht, sht, k16_off(row, 0), &shv[0]);
                store_chunk<false, false>(sht, sht, k16_off(row, 1), &shv[8]);
                newray = false;
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                *reinterpret_cast<uint4 *>(h + sw128_off(row, c)) = pos_chunk(c);
                if (ROBUST) *reinterpret_cast<uint4 *>(l + sw128_off(row, c)) = make_uint4(featl[4 * c], featl[4 * c + 1], featl[4 * c + 2], featl[4 * c + 3]);
            }
            {   // the frame's conditioning vector as pre-rounded fp16 images (k_cond_images): 8 x 16 bytes straight into the operand tiles
                const uint4 *ch = reinterpret_cast<const uint4 *>(t.cond_hi) + (size_t)cu.frame * 8;
                const uint4 *cl = reinterpret_cast<const uint4 *>(t.cond_lo) + (size_t)cu.frame * 8;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const uint32_t off = (c < 4) ? sw128_off(row, 4 + c) : (uint32_t)V2_TILE_BYTES + sw128_off(row, c - 4);
                    *reinterpret_cast<uint4 *>(h + off) = __ldg(ch + c);
                    if (ROBUST) *reinterpret_cast<uint4 *>(l + off) = __ldg(cl + c);
                }
            }
            PH(0)   // operand rows of ambient L0

            // ---------------- fate of the ray, march to the next sample, refill (the other slots' MMAs run meanwhile) ----------------
            if (valid) {
                const int ns = cu.nsamp + 1;                 // samples composited once this one is
                const float T = 1.0f - cu.ws;
                if (T < a.T_thresh) { cu.fate = 1; cu.D = ns; }
                else if (ns >= sl.cap) cu.fate = 2;
                else if (!march_next(mc, sl.g, sl.far_m, sl.t, sl.px, sl.py, sl.pz, sl.dt)) { cu.fate = 1; cu.D = ns + 1; }
                else { cu.fate = 0; sl.nsamp = ns; }
                if (cu.fate) sl.active = false;
            }
            __syncwarp();
            refill();
            PH(1)   // fate + march + refill
            ARRIVE_A();   // -> ambient L0

            // ---------------- ambient net 96 -> 128 -> 128 -> 3 (radnerf.py:121) ----------------
            // one 128-wide ambient layer: two K tiles (ks0, ks1 k-steps), in the robust mode each as (hi, lo) weight images and
            // D = Al*Wh + Ah*Wl + Ah*Wh, small terms first
            auto amb_layer = [&](int ks0, int ks1) {
                uint32_t wt[ROBUST ? 4 : 2];
#pragma unroll
                for (int j = 0; j < (ROBUST ? 4 : 2); ++j) wt[j] = tile((uint32_t)j);
#pragma unroll 1
                for (int hf = 0; hf < 2; ++hf) {
                    const uint32_t o = (uint32_t)hf * SW128_HALF;
                    float d[64];
                    wg_fence();
                    if (ROBUST) {
#pragma unroll
                        for (int kt = 0; kt < 2; ++kt) {
                            const uint32_t wh = wt[ROBUST ? 2 * kt : 0], wl = wt[ROBUST ? 2 * kt + 1 : 0], tk = (uint32_t)kt * V2_TILE_BYTES + o;
                            const int ks = kt ? ks1 : ks0;
                            wgmma_sw<128, false>(d, l_u + tk, wh, ks, kt ? 1u : 0u);
                            wgmma_sw<128, false>(d, h_u + tk, wl, ks, 1u);
                            wgmma_sw<128, false>(d, h_u + tk, wh, ks, 1u);
                        }
                    } else {
                        wgmma_sw<128, false>(d, h_u + o, wt[0], ks0, 0u);
                        wgmma_sw<128, false>(d, h_u + V2_TILE_BYTES + o, wt[1], ks1, 1u);
                    }
                    wg_commit();
                    wg_wait<0>();
                    acc_fence(d);
                    epilogue_half<true, false, ROBUST>(d, h, l, hf, lane, wwarp, nullptr);
                }
                release(ROBUST ? 4 : 2);
            };
            amb_layer(4, 2);   // ambient L0: K = 96 = 32 position features + 64 conditioning values (h0 k[0,64), h1 k[0,32))
            ARRIVE_A();   // -> ambient L1
            PH(2)   // MMA + epilogue: ambient L0
            amb_layer(4, 4);   // ambient L1: K = 128
            ARRIVE_A();   // -> ambient out (N = 16)
            PH(3)   // MMA + epilogue: ambient L1
#pragma unroll 1
            for (int hf = 0; hf < 2; ++hf) {   // ambient out: N = 16 group from the resident tiles
                const uint32_t o = (uint32_t)hf * SW128_HALF;
                float d[8];
                wg_fence();
                if (ROBUST) {
                    mma16(d, l_u + o, res_u + V2_RES_AMBN_HI, 0u);
                    mma16(d, h_u + o, res_u + V2_RES_AMBN_LO, 1u);
                }
                mma16(d, h_u + o, res_u + V2_RES_AMBN_HI, ROBUST ? 1u : 0u);
                wg_commit();
                wg_wait<0>();
                acc_fence(d);
                put_cols<3>(d, outc, 0, hf, lane, wwarp);
            }
            wg_sync(1 + s);
            PH(4)   // MMA: ambient out
            const float amb0 = tanhf(outc[row]), amb1 = tanhf(outc[TM + row]), amb2 = tanhf(outc[2 * TM + row]);
            PH(5)   // tanh
            // ---------------- sigma-net input: h0 k[0,32) <- position features, k[32,64) <- ambient grid ----------------
            {
                float u = 0.f, vv = 0.f, w = 0.f;
                if (valid) {   // GridEncoder.forward with bound = 1: (x + 1) / 2
                    u = __fdiv_rn(__fadd_rn(amb0, 1.0f), 2.0f);
                    vv = __fdiv_rn(__fadd_rn(amb1, 1.0f), 2.0f);
                    w = __fdiv_rn(__fadd_rn(amb2, 1.0f), 2.0f);
                }
#pragma unroll
                for (int c = 0; c < 4; ++c) *reinterpret_cast<uint4 *>(h + sw128_off(row, c)) = pos_chunk(c);
                // that was the last read of the staging row: it takes the next request now, so the gather warp's lookups run in the
                // shadow of the ambient gather and this slot's sigma and colour nets
                if (C::STAGED) post_pos();
#pragma unroll 1
                for (int half = 0; half < 2; ++half) {
                    float f[16];
                    if (valid) {
                        lookup8<OCT_F16>(&ms.lvl[1][half * 16], a.amb_gm.align_off, smooth_a, a.amb_octs, u, vv, w, f);
                    } else {
#pragma unroll
                        for (int i = 0; i < 16; ++i) f[i] = 0.f;
                    }
                    store_chunk<false, false>(h, h, sw128_off(row, 4 + 2 * half), &f[0]);
                    store_chunk<false, false>(h, h, sw128_off(row, 4 + 2 * half + 1), &f[8]);
                }
            }
            PH(7)   // ambient gather
            // the NEXT sample's position features the owner looks up itself (the current ones are in the operand tile now)
            if (C::OWN_LV > 0) {
                prefetch_pos(0);
                PH(8)   // prefetch: position levels 0-7 of the next sample
            }
            ARRIVE_A();   // -> sigma L0

            // ---------------- sigma net 64 -> 128 -> 128 -> (128 geo + sigma) (radnerf.py:127-130) ----------------
            layer128(1, [&](float (&d)[64], uint32_t o, uint32_t w0, uint32_t) { wgmma_sw<128, false>(d, h_u + o, w0, 4, 0u); },   // sigma L0: K = 64
                     [&](const float (&d)[64], int hf) { epilogue_half<true, false, false>(d, h, h, hf, lane, wwarp, nullptr); });
            ARRIVE_A();   // -> sigma L1
            PH(9)   // MMA + epilogue: sigma L0
            if (C::OWN_LV > 8) {
                prefetch_pos(1);
                PH(10)  // prefetch: position levels 8-15 of the next sample
            }
            layer128(2, [&](float (&d)[64], uint32_t o, uint32_t w0, uint32_t w1) {   // sigma L1: K = 128
                wgmma_sw<128, false>(d, h_u + o, w0, 4, 0u);
                wgmma_sw<128, false>(d, h_u + V2_TILE_BYTES + o, w1, 4, 1u);
            }, [&](const float (&d)[64], int hf) { epilogue_half<true, false, false>(d, h, h, hf, lane, wwarp, nullptr); });
            ARRIVE_A();   // -> color L0 + sigma row
            PH(11)  // MMA + epilogue: sigma L1

            // ---------------- sigma L2 + color net (16 SH + 128 geo [+ folded individual code]) -> 128 -> 3 (radnerf.py:127-141) ----------------
            // The 128 geo rows of sigma L2 have no activation and only feed color L0, which is linear in them: the pack folds them into
            // color L0's geo columns (W_fold = W_c0[:, 16:144] * W_s2[1:129, :], k_pack_fold_tile), so color L0 reads sigma L1's output
            // h_s1 directly.  One commit group per M-half: W_fold over K = 128 (streamed), SH K = 16 (resident no-swizzle tile against
            // the slot's SH operand tile), and the sigma row of sigma L2 (resident N = 16 tile) on the same h_s1 operand rows.
            {
                const uint32_t w0 = tile(0), w1 = tile(1);
#pragma unroll 1
                for (int hf = 0; hf < 2; ++hf) {
                    const uint32_t o = (uint32_t)hf * SW128_HALF;
                    float d[64], d16[8];
                    wg_fence();
                    wgmma_sw<128, false>(d, h_u + o, w0, 4, 0u);
                    wgmma_sw<128, false>(d, h_u + V2_TILE_BYTES + o, w1, 4, 1u);
                    wgmma<128, false>(d, desc_k16(sh_u + (o ? K16_HALF : 0u)), desc_k16(res_u + V2_RES_COLSH), 1u);
                    mma16(d16, h_u + o, res_u + V2_RES_SIGROW, 0u);
                    wg_commit();
                    wg_wait<0>();
                    acc_fence(d);
                    acc_fence(d16);
                    if ((lane & 3) == 0) {   // the sigma logit (column 0) of fragment rows r, r+8
                        slogit[64 * hf + frag_row(0, lane, wwarp)] = d16[0];
                        slogit[64 * hf + frag_row(2, lane, wwarp)] = d16[2];
                    }
                    epilogue_half<true, true, false>(d, h, h, hf, lane, wwarp, ms.cbias);
                }
                release(2);
            }
            ARRIVE_A();   // -> color out (N = 16)
            PH(13)  // MMA + epilogue: sigma row + color L0
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {   // color out: N = 16 group -> the hand-over buffer
                const uint32_t o = (uint32_t)hf * SW128_HALF;
                float d[8];
                wg_fence();
                mma16(d, h_u + o, res_u + V2_RES_COLN, 0u);
                wg_commit();
                wg_wait<0>();
                acc_fence(d);
                put_cols<3>(d, outc, 0, hf, lane, wwarp);
            }
            wg_sync(1 + s);
            PH(14)  // MMA: color out
            // trunc_exp forward (utils.py:36-49) * density_scale (renderer.py:365)
            const float sigma = a.density_scale * expf(slogit[row]);
            const float cr = 1.0f / (1.0f + expf(-outc[row]));
            const float cg = 1.0f / (1.0f + expf(-outc[TM + row]));
            const float cb = 1.0f / (1.0f + expf(-outc[2 * TM + row]));
            wg_sync(1 + s);   // the next batch's operand rows overwrite the hand-over buffer
            PH(15)  // sigmoid

            // ---------------- composite the sample (raymarching.cu:978-1006) and retire / suspend / continue its ray ----------------
            if (valid) {
                const float alpha = 1.0f - expf(-sigma * cu.dt);
                const float T = 1.0f - cu.ws;
                const float wgt = alpha * T;
                cu.ws += wgt;
                cu.depth += wgt * cu.t_post;   // deltas[1]: t after the sample
                cu.r += wgt * cr;
                cu.g += wgt * cg;
                cu.b += wgt * cb;
                if (a.valid_samples) warp_agg_add(a.valid_samples, cu.frame, 1);
                if (cu.fate == 0) {            // same ray goes on: `sl` (already at its next sample) takes the accumulators
                    sl.ws = cu.ws; sl.depth = cu.depth; sl.r = cu.r; sl.gch = cu.g; sl.b = cu.b;
                } else {
                    const size_t g = (size_t)cu.gid;
                    const bool normalise = cu.fate == 1 || a.pass != 1;   // a suspended pass-1 ray keeps its raw depth: pass 2 goes on accumulating
                    a.image[3 * g] = cu.r; a.image[3 * g + 1] = cu.g; a.image[3 * g + 2] = cu.b;
                    a.wsum[g] = cu.ws;
                    // renderer.py:394: depth = clamp(depth - nears, min=0) / (fars - nears)
                    a.depth[g] = normalise ? __fdiv_rn(fmaxf(__fsub_rn(cu.depth, cu.near), 0.f), __fsub_rn(cu.far, cu.near)) : cu.depth;
                    if (cu.fate == 1) {
                        if (a.pass == 1) warp_agg_add(a.hist, cu.frame * (a.max_steps + 2) + cu.D, 1);
                    } else if (a.pass == 1) {
                        a.rays_t[g] = cu.t_post;
                        cg::coalesced_group grp = cg::coalesced_threads();
                        int base = 0;
                        if (grp.thread_rank() == 0) base = atomicAdd(a.n_survivors, (int)grp.size());
                        base = grp.shfl(base, 0);
                        a.survivors[base + grp.thread_rank()] = cu.gid;
                    }
                }
            }
            __syncwarp();
            rotate();

            // ---------------- end of batch: was anything alive in it? ----------------
            mbar_wait(&ms.batch_bar, bpar);
            int any = 0;
#pragma unroll
            for (int i = 0; i < NWORK; ++i) any |= ms.flag[bpar][i];
            bpar ^= 1u;
            __syncwarp();
            PH(19)  // composite + end-of-batch check
            if (PROFILE && a.phase_cycles && tid == 0) atomicAdd(a.phase_cycles + 31, 1ull);   // batches
            if (!any) break;
        }
#undef PH
#undef ARRIVE_A
        if (C::STAGED) {   // once the gather warp has served the last batch's request, a final one with the quit flag releases it
            mbar_wait(&ms.pos_done[s], bpar);
            if (row == 0) ms.pos_quit[s] = 1;
            mbar_arrive(&ms.pos_req[s]);
        }
        // stop the loader: the NSTAGE tiles it has prefetched for a batch that never comes must land before the CTA may exit.
        // `stop` is raised only once all of them have landed: the other slots may still be releasing their last tiles, and a
        // loader that saw `stop` before issuing these would leave the waits below hanging.
#pragma unroll 1
        for (uint32_t j = 0; j < (uint32_t)NSTAGE; ++j) mbar_wait(&ms.w_full[(wc + j) % NSTAGE], ((wc + j) / NSTAGE) & 1u);
        if (lane == 0) {
            ms.stop = 1;
            __threadfence_block();
            for (uint32_t j = 0; j < (uint32_t)NSTAGE; ++j) mbar_arrive(&ms.w_free[(wc + j) % NSTAGE]);
        }
        __syncwarp();
    } else {
        // =====================================================================================================
        // PRODUCER WARPGROUP: hands its registers to the owners; warp 0 is the LOADER, warp 1 + s (fp16) the GATHER WARP of
        // slot s, any other leaves.  `w_free` and `batch_bar` count owner warps, the named barriers the 128 threads of one slot;
        // only `pos_done` counts a gather warp, and its owners stop waiting on it before they release it.
        // =====================================================================================================
        setmaxnreg_dec<C::PRODUCER_REGS>();
        if (C::STAGED && warp > NWORK && warp <= NWORK + C::NSLOT) {
            // GATHER WARP: per request of its slot, the 16 - GATHER_L0 position levels [GATHER_L0, 16) of every row's posted point
            // into the row's staging slot; lane l serves rows l, l + 32, .., GATHER_N levels per lookup call
            const int gs = warp - NWORK - 1;
            unsigned char *sg = stage + gs * TM * 64;
            const bool smooth = a.pos_gm.interp == 1;
#pragma unroll 1
            for (uint32_t par = 0;; par ^= 1u) {
                mbar_wait(&ms.pos_req[gs], par);
                if (ms.pos_quit[gs]) break;
                // outside the grid the lookup gives zeros (gather8.cuh): its loads are skipped
                auto inside = [](const float4 &p) { return !(p.x < 0.f || p.x > 1.f || p.y < 0.f || p.y > 1.f || p.z < 0.f || p.z > 1.f); };
                // a row's octs go towards L2 one row ahead of its loads: GATHER_N loads in flight per lane are too few to cover
                // DRAM latency on their own
                auto prefetch_row = [&](int r) {
                    const float4 p = *reinterpret_cast<const float4 *>(sg + stage_off(r, GATHER_L0 / 4));
                    if (inside(p)) prefetch_levels_l2<16 - GATHER_L0>(&ms.lvl[0][2 * GATHER_L0], a.pos_gm.align_off, a.pos_octs, p.x, p.y, p.z);
                };
                prefetch_row(lane);
#pragma unroll 1
                for (int r = lane; r < TM; r += 32) {
                    const float4 p = *reinterpret_cast<const float4 *>(sg + stage_off(r, GATHER_L0 / 4));
                    const bool in = inside(p);
                    if (r + 32 < TM) prefetch_row(r + 32);
#pragma unroll 1
                    for (int lv = GATHER_L0; lv < 16; lv += GATHER_N) {
                        float f[2 * GATHER_N];
                        if (in) {
                            lookup_levels<OCT_F16, GATHER_N>(&ms.lvl[0][2 * lv], a.pos_gm.align_off, smooth, a.pos_octs, p.x, p.y, p.z, f);
                        } else {
#pragma unroll
                            for (int i = 0; i < 2 * GATHER_N; ++i) f[i] = 0.f;
                        }
                        uint32_t q[GATHER_N];
#pragma unroll
                        for (int i = 0; i < GATHER_N; ++i) q[i] = pack2<false>(f[2 * i], f[2 * i + 1]);
#pragma unroll
                        for (int i = 0; i < GATHER_N; i += 2)   // level lv + i in word (lv + i) % 4 of chunk (lv + i) / 4
                            *reinterpret_cast<uint2 *>(sg + stage_off(r, (lv + i) / 4) + 4 * ((lv + i) % 4)) = make_uint2(q[i], q[i + 1]);
                    }
                }
                mbar_arrive(&ms.pos_done[gs]);
            }
            return;
        }
        if (warp != NWORK) return;
        // LOADER: resident tiles once, then the weight stream, NSTAGE tiles ahead of the issue warp
        if (elect_one()) {
            mbar_expect_tx(&ms.res_full, V2_RES_BYTES);
            bulk_g2s(res, t.w_res, V2_RES_BYTES, &ms.res_full);
        }
        __syncwarp();
        for (uint32_t i = 0;; ++i) {
            const uint32_t stage = i % NSTAGE;
            if (i >= (uint32_t)NSTAGE) mbar_wait(&ms.w_free[stage], ((i / NSTAGE) - 1u) & 1u);
            if (ms.stop) break;
            if (elect_one()) {
                mbar_expect_tx(&ms.w_full[stage], V2_TILE_BYTES);
                bulk_g2s(wring + stage * V2_TILE_BYTES, t.w_stream + (size_t)(i % NTILE) * V2_TILE_BYTES, V2_TILE_BYTES, &ms.w_full[stage]);
            }
            __syncwarp();
        }
    }

}

size_t head_v2_smem_bytes(bool robust) { return robust ? smem_bytes<true>() : smem_bytes<false>(); }

cudaError_t launch_cond_images(const float *cond_feat, int n_frames, void *cond_hi, void *cond_lo, cudaStream_t st) {
    const int n = n_frames * 64;
    k_cond_images<<<(n + 255) / 256, 256, 0, st>>>(cond_feat, n, (__half *)cond_hi, (__half *)cond_lo);
    return cudaGetLastError();
}

cudaError_t launch_head_v2(const HeadArgs &a, const HeadV2Args &t_in, int precision, cudaStream_t st) {
    const HeadV2Args &t = t_in;
    const bool robust = precision == FP16_ROBUST;
    if (!robust && precision != FP16_X1) return cudaErrorInvalidValue;
    const int blocks = sm_count();   // persistent: one CTA per SM (~200 KB of shared memory each)
    const size_t smem = head_v2_smem_bytes(robust);
    cudaError_t e;
    // function attributes are per device: set on every launch.  The phase-stamped instantiation only runs under tools/phase_breakdown.py.
#define GO(RB, PF)                                                                                                   \
    e = cudaFuncSetAttribute(k_head_v2<RB, PF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);             \
    if (e != cudaSuccess) return e;                                                                                  \
    k_head_v2<RB, PF><<<blocks, Cfg<RB>::NT, smem, st>>>(a, t);
    if (robust) { if (a.phase_cycles) { GO(true, true) } else { GO(true, false) } }
    else { if (a.phase_cycles) { GO(false, true) } else { GO(false, false) } }
#undef GO
    return cudaGetLastError();
}

}  // namespace gfpp
