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
//   * the narrow layers (ambient out, colour out; K = 128, N = 3) run in the epilogue of the layer that feeds them: per warp,
//     eight chained mma.sync m16n8k16 whose A fragments are that layer's accumulator registers after ReLU and fp16 rounding,
//     against per-lane B-fragment images in the RESIDENT block -- no operand-tile store, no async proxy, no wgmma round trip.
//     The sigma row of sigma L2 (N = 1) reads sigma L1's stored output back with ldmatrix while color L0's MMAs run.  Their
//     columns go to the row owners through a small buffer at the head of the slot's second operand tile (ambient out) and a
//     per-row buffer (sigma logit, colour out);
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

// the sigma logits and color out of a slot's rows, from their mma.sync (under / in color L0) to the row owners, [4][TM] floats per
// slot (sigma, r, g, b): the robust mode keeps them at the head of the slot's residual tile l (idle from ambient L1's MMA to the
// next batch's operand rows), fp16 behind Misc
template <bool ROBUST>
constexpr size_t slogit_bytes() { return ROBUST ? 0 : (size_t)Cfg<ROBUST>::NSLOT * 4 * TM * sizeof(float); }
// fp16: the gather warps' staging rows behind the sigma logits, [NSLOT][TM] x 64 bytes: 16 levels as packed fp16 pairs (level j
// in 32-bit word j) or, from the owner's post to the gather warp's reply, the row's next grid coordinates in chunk 0
template <bool ROBUST>
constexpr size_t stage_bytes() { return Cfg<ROBUST>::STAGED ? (size_t)Cfg<ROBUST>::NSLOT * TM * 64 : 0; }
template <bool ROBUST>
constexpr size_t smem_bytes() { return (size_t)Cfg<ROBUST>::OFF_MISC + sizeof(Misc) + slogit_bytes<ROBUST>() + stage_bytes<ROBUST>() + 1024; }
static_assert(smem_bytes<false>() <= 227 * 1024 && smem_bytes<true>() <= 227 * 1024, "v2 shared memory budget");

// Epilogue of one M = 64 half (rows 64*half ..) of a 128-wide layer from the accumulator fragment: (+bias) -> (ReLU) ->
// operand tiles h0|h1 (cols 0-63 | 64-127) and, when LO, the residual images l0|l1.  BIAS: shared-memory vector (color L0).
// Without LO the pairs of two 8-column blocks go out in one stmatrix: 8 stores per thread instead of 32.
template <bool RELU, bool BIAS, bool LO>
__device__ __forceinline__ void epilogue_half(const float (&d)[64], unsigned char *h, unsigned char *l, int half, int lane, int wwarp,
                                              const float *bias) {
    if constexpr (LO) {
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int row = 64 * half + frag_row(i, lane, wwarp), col = frag_col(i, lane);
            float x0 = d[i], x1 = d[i + 1];
            if (BIAS) { x0 += bias[col]; x1 += bias[col + 1]; }
            if (RELU) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            store_pair<false, LO>(h + (col >> 6) * V2_TILE_BYTES, l + (col >> 6) * V2_TILE_BYTES, row, col & 63, x0, x1);
        }
    } else {
        // matrix j of a store is the 8 x 8 block of rows +8 (j & 1), column block cb + (j >> 1): fragment pairs 4 cb + 2 j, +1.
        // Lane l addresses row l % 8 of matrix l / 8
        const int m = lane >> 3, arow = 64 * half + 16 * wwarp + 8 * (m & 1) + (lane & 7);
        const uint32_t h_u = smem_u32(h);
#pragma unroll
        for (int cb = 0; cb < 16; cb += 2) {
            uint32_t q[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * cb + 2 * j, col = frag_col(i, lane);
                float x0 = d[i], x1 = d[i + 1];
                if (BIAS) { x0 += bias[col]; x1 += bias[col + 1]; }
                if (RELU) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                q[j] = pack2<false>(x0, x1);
            }
            const int c = cb + (m >> 1);
            stmatrix_x4(h_u + (uint32_t)(c >> 3) * V2_TILE_BYTES + sw128_off(arow, c & 7), q[0], q[1], q[2], q[3]);
        }
    }
}

// The store of epilogue_half<.., .., false> from an image relu_pack made: the pairs of column blocks cb, cb + 1 are a[2cb .. 2cb + 3]
__device__ __forceinline__ void store_half(const uint32_t (&a)[32], unsigned char *h, int half, int lane, int wwarp) {
    const int m = lane >> 3, arow = 64 * half + 16 * wwarp + 8 * (m & 1) + (lane & 7);
    const uint32_t h_u = smem_u32(h);
#pragma unroll
    for (int cb = 0; cb < 16; cb += 2) {
        const int c = cb + (m >> 1);
        stmatrix_x4(h_u + (uint32_t)(c >> 3) * V2_TILE_BYTES + sw128_off(arow, c & 7), a[2 * cb], a[2 * cb + 1], a[2 * cb + 2], a[2 * cb + 3]);
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

// The fp16 operand image of a warp's rows of a 128-wide layer, from its accumulator fragment: (+bias) -> ReLU -> a[m] = the
// rounded pair (d[2m], d[2m + 1]), exactly the values the epilogue stores; a[4kb .. 4kb + 3] is the mma.sync A fragment of
// k-block kb.  LO: al[m] = the residual pair, x - rn16(x), as store_pair<false, true> writes it.
template <bool BIAS, bool LO>
__device__ __forceinline__ void relu_pack(const float (&d)[64], const float *bias, int lane, uint32_t (&a)[32], uint32_t (&al)[LO ? 32 : 1]) {
#pragma unroll
    for (int m = 0; m < 32; ++m) {
        const int col = frag_col(2 * m, lane);
        float x0 = d[2 * m], x1 = d[2 * m + 1];
        if (BIAS) { x0 += bias[col]; x1 += bias[col + 1]; }
        x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f);
        a[m] = pack2<false>(x0, x1);
        if constexpr (LO) al[m] = pack2<false>(x0 - round16<false>(x0), x1 - round16<false>(x1));
    }
}

// A narrow layer (K = 128, N <= 8) on one warp's 16 rows: c (+)= A[16 x 128] * B[128 x 8], eight mma.sync in k order, the A
// fragments from relu_pack, B from the per-lane fragment image at `img` (k_pack_narrow_b): the sum order of the N = 16 wgmma
// chain it replaces.  ACC = false starts from zero
template <bool ACC>
__device__ __forceinline__ void narrow_mma(float (&c)[4], const uint32_t (&a)[32], const unsigned char *img, int lane) {
    if (!ACC) c[0] = c[1] = c[2] = c[3] = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 b = *reinterpret_cast<const uint4 *>(img + q * 512 + lane * 16);
        mma_m16n8k16(c, a[8 * q], a[8 * q + 1], a[8 * q + 2], a[8 * q + 3], b.x, b.y);
        mma_m16n8k16(c, a[8 * q + 4], a[8 * q + 5], a[8 * q + 6], a[8 * q + 7], b.z, b.w);
    }
}

// The narrow layer of narrow_mma with A read back from the operand tiles h0|h1 that store_half wrote (rows of warp `wwarp`,
// M-half `half`), one k-block at a time with ldmatrix: the same fp16 values, and no image held in registers
__device__ __forceinline__ void narrow_mma_smem(float (&c)[4], const unsigned char *h, int half, const unsigned char *img, int lane, int wwarp) {
    const int m = lane >> 3, arow = 64 * half + 16 * wwarp + 8 * (m & 1) + (lane & 7);
    const uint32_t h_u = smem_u32(h);
    c[0] = c[1] = c[2] = c[3] = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 b = *reinterpret_cast<const uint4 *>(img + q * 512 + lane * 16);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int ch = 4 * q + 2 * j + (m >> 1);   // 16-byte chunk of k-block 2q + j this lane addresses
            uint32_t a0, a1, a2, a3;
            ldmatrix_x4(h_u + (uint32_t)(ch >> 3) * V2_TILE_BYTES + sw128_off(arow, ch & 7), a0, a1, a2, a3);
            mma_m16n8k16(c, a0, a1, a2, a3, j ? b.z : b.x, j ? b.w : b.y);
        }
    }
}

// Columns 0 .. NC-1 of a narrow product (m16n8 D fragment of warp `wwarp`, M-half `half`) -> out[c][row], read back by the row
// owners: lane 4g + t holds rows g and g + 8 at columns 2t and 2t + 1
template <int NC>
__device__ __forceinline__ void put_cols(const float (&c)[4], float *out, int half, int lane, int wwarp) {
    const int col = 2 * (lane & 3), row = 64 * half + 16 * wwarp + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 2; ++j)
        if (col + j < NC) { out[(col + j) * TM + row] = c[j]; out[(col + j) * TM + row + 8] = c[2 + j]; }
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
    constexpr bool TRAIN = false;
#include "head_v2_body.inc"
}

template <bool ROBUST>
__global__ void __launch_bounds__(Cfg<ROBUST>::NT, 1) k_head_v2_train(const __grid_constant__ HeadArgs a, const __grid_constant__ HeadV2Args t) {
    constexpr bool PROFILE = false, TRAIN = true;
#include "head_v2_body.inc"
}

size_t head_v2_smem_bytes(bool robust) { return robust ? smem_bytes<true>() : smem_bytes<false>(); }

cudaError_t launch_cond_images(const float *cond_feat, int n_frames, void *cond_hi, void *cond_lo, cudaStream_t st) {
    const int n = n_frames * 64;
    k_cond_images<<<(n + 255) / 256, 256, 0, st>>>(cond_feat, n, (__half *)cond_hi, (__half *)cond_lo);
    return cudaGetLastError();
}

cudaError_t launch_head_v2(const HeadArgs &a, const HeadV2Args &t_in, int precision, cudaStream_t st, bool train) {
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
#define GO_TRAIN(RB)                                                                                                 \
    e = cudaFuncSetAttribute(k_head_v2_train<RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);           \
    if (e != cudaSuccess) return e;                                                                                  \
    k_head_v2_train<RB><<<blocks, Cfg<RB>::NT, smem, st>>>(a, t);
    if (train) { if (robust) { GO_TRAIN(true) } else { GO_TRAIN(false) } }
    else if (robust) { if (a.phase_cycles) { GO(true, true) } else { GO(true, false) } }
    else { if (a.phase_cycles) { GO(false, true) } else { GO(false, false) } }
#undef GO_TRAIN
#undef GO
    return cudaGetLastError();
}

}  // namespace gfpp
