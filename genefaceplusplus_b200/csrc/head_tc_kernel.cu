// head_tc_kernel.cu -- fused persistent head renderer, tensor-core variant (wgmma + TMA bulk copies).
//
// Same ray-slot machinery, marching, gather and compositing as head_kernel.cu; only the dense tiny-MLP GEMMs differ:
// every 128-row batch runs its eight layers as wgmma.mma_async (16-bit operands, fp32 accumulate, N in {128,144}), the
// two warpgroups of the CTA taking rows 0-63 and 64-127, with
//   * A (activations) written by the CTA's threads straight into GMMA K-major SW128 tiles in shared memory
//     (gathered grid features, conditioning, previous layer's epilogue), 16-bit, optionally hi/lo split;
//   * W streamed as pre-swizzled 16-bit tiles through a 3-stage ring with cp.async.bulk + mbarrier;
//   * D (fp32 accumulators) in registers, consumed in the accumulator fragment layout by the ReLU / tanh / exp /
//     sigmoid epilogues;
//   * position-grid features parked in registers (their 16-bit operand chunks) between the ambient and sigma nets.
//
// Precision modes (tc::Precision): FP16_X1 (what the reference itself runs under autocast, fp32 accumulate),
// BF16_X1, BF16_X3 (hi/lo split, 3 MMAs per k-step: ~16 mantissa bits).  See DESIGN.md "precision".
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

constexpr int TM = HEAD_TM;
constexpr int NT = HEAD_NT;
constexpr int A_TILE = 16384;        // 128 rows x 64 k x 2 B (SW128)
constexpr int A_K16 = 4096;          // 128 rows x 16 k x 2 B (no swizzle)
constexpr int W_HALF = 18432;        // up to 144 rows x 64 k x 2 B
constexpr int W_NSTAGE = 3;

// the lo (split) operand images exist only in the bf16x3 instantiation; the single-pass kernels stay under 113 KB of
// shared memory and 128 registers so that TWO CTAs are resident per SM (their barrier / latency stalls overlap)
template <bool SPLIT>
struct SmemTC {
    // SW128 tiles must start on 1024-byte boundaries (the swizzle is a function of the shared-memory address bits)
    alignas(1024) unsigned char a_hi[2][A_TILE];
    alignas(1024) unsigned char w_hi[W_NSTAGE][W_HALF];
    alignas(SPLIT ? 1024 : 16) unsigned char a_lo[SPLIT ? 2 : 1][SPLIT ? A_TILE : 16];
    alignas(SPLIT ? 1024 : 16) unsigned char w_lo[SPLIT ? W_NSTAGE : 1][SPLIT ? W_HALF : 16];
    alignas(256) unsigned char s_hi[A_K16];
    alignas(SPLIT ? 256 : 16) unsigned char s_lo[SPLIT ? A_K16 : 16];
    float bias[128];                  // color L0 bias (individual code folded)
    float nw[6 * 128];                // fp32 rows of the two 3-wide output layers: ambient out (0-2), color out (3-5)
    float part[3 * TM];               // their dot products
    float sx[TM], sy[TM], sz[TM];
    float amb[3 * TM];
    float sig[TM];
    float rgb[3 * TM];
    int frame[TM];
    int valid[TM];
    unsigned long long bar_full[W_NSTAGE];
    uint32_t coarse[HEAD_COARSE_WORDS];
    uint4 lvl[2][2 * GFPP_MAX_LEVELS];   // per-level grid metadata (position, ambient) for lookup8o
    int next, end, done;
};

// The weight stream is static: batch b consumes tiles b*12 + (0..11) in the order of kHeadTcChunks, and 12 is a multiple
// of the ring depth, so tile id c always lives in stage c % W_NSTAGE and completes the mbarrier phase (c / W_NSTAGE) & 1.
static_assert(HEAD_TC_NCHUNK % W_NSTAGE == 0, "the static stage/parity schedule needs the ring depth to divide the tiles per batch");

template <bool SPLIT, int ID>
__device__ __forceinline__ void issue_load(const HeadTcArgs &t, SmemTC<SPLIT> &s) {
    constexpr int id = ID % HEAD_TC_NCHUNK, stage = id % W_NSTAGE;
    constexpr uint32_t bytes = (uint32_t)head_tc_chunk_bytes(id), off = (uint32_t)head_tc_chunk_off(id);
    mbar_expect_tx(&s.bar_full[stage], SPLIT ? 2 * bytes : bytes);
    bulk_g2s(s.w_hi[stage], t.w_hi + off, bytes, &s.bar_full[stage]);
    if (SPLIT) bulk_g2s(s.w_lo[SPLIT ? stage : 0], t.w_lo + off, bytes, &s.bar_full[stage]);
}
template <bool SPLIT, int ID, int N>
__device__ __forceinline__ void issue_loads(const HeadTcArgs &t, SmemTC<SPLIT> &s) {
    if constexpr (N > 0) {
        issue_load<SPLIT, ID>(t, s);
        issue_loads<SPLIT, ID + 1, N - 1>(t, s);
    }
}

// the MMAs of tile ID against A tile `a_tile` (the K16 SH tile for the k16 chunk), rows of warpgroup `wg`
template <bool BF16, bool SPLIT, int ID, bool ACC0, int N>
__device__ __forceinline__ void mma_tile(SmemTC<SPLIT> &s, int a_tile, int wg, float (&d)[N / 2]) {
    constexpr int stage = ID % W_NSTAGE, ksteps = head_tc_chunk_ksteps(ID);
    constexpr bool k16 = kHeadTcChunks[ID].k16 != 0;
    const uint32_t half = (uint32_t)wg * (k16 ? K16_HALF : SW128_HALF);
    const uint32_t ah = (k16 ? smem_u32(s.s_hi) : smem_u32(s.a_hi[a_tile])) + half;
    const uint32_t al = (k16 ? smem_u32(s.s_lo) : smem_u32(s.a_lo[SPLIT ? a_tile : 0])) + half;
    const uint32_t wh = smem_u32(s.w_hi[stage]), wl = smem_u32(s.w_lo[SPLIT ? stage : 0]);
#pragma unroll
    for (int k = 0; k < ksteps; ++k) {
        const uint32_t adv = (uint32_t)k * 32u;   // 16 elements x 2 B inside the 128-byte swizzle row
        const uint64_t dah = k16 ? desc_k16(ah) : desc_sw128(ah + adv), dwh = k16 ? desc_k16(wh) : desc_sw128(wh + adv);
        const uint32_t acc0 = (ACC0 || k > 0) ? 1u : 0u;
        if (SPLIT) {
            const uint64_t dal = k16 ? desc_k16(al) : desc_sw128(al + adv), dwl = k16 ? desc_k16(wl) : desc_sw128(wl + adv);
            wgmma<N, BF16>(d, dal, dwh, acc0);   // small terms first
            wgmma<N, BF16>(d, dah, dwl, 1u);
            wgmma<N, BF16>(d, dah, dwh, 1u);
        } else {
            wgmma<N, BF16>(d, dah, dwh, acc0);
        }
    }
}
template <bool BF16, bool SPLIT, int ID, int C, int NCH, int N>
__device__ __forceinline__ void mma_tiles(SmemTC<SPLIT> &s, int wg, float (&d)[N / 2]) {
    if constexpr (C < NCH) {
        mma_tile<BF16, SPLIT, ID, (C > 0), N>(s, C, wg, d);
        mma_tiles<BF16, SPLIT, ID + 1, C + 1, NCH, N>(s, wg, d);
    }
}

// One layer = tiles ID0 .. ID0+NCH-1 against A tiles 0,1,.. for the 64 rows of the calling warpgroup; returns with the
// accumulators complete.  Then (CTA barrier: both warpgroups are done with the weight stages) warp 0 refills the stages.
template <bool BF16, bool SPLIT, int ID0, int NCH, int N>
__device__ __forceinline__ void mma_layer(const HeadTcArgs &t, SmemTC<SPLIT> &s, int wg, int warp, float (&d)[N / 2]) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) mbar_wait(&s.bar_full[(ID0 + c) % W_NSTAGE], ((ID0 + c) / W_NSTAGE) & 1);
    wg_fence();
    mma_tiles<BF16, SPLIT, ID0, 0, NCH, N>(s, wg, d);
    wg_commit();
    wg_wait<0>();
    acc_fence(d);
    __syncthreads();
    if (warp == 0) {
        if (elect_one()) issue_loads<SPLIT, ID0 + W_NSTAGE, NCH>(t, s);
        __syncwarp();
    }
}

// Epilogue of a 128-wide layer from the accumulator fragment (columns 0..127 of d): bias/ReLU, then either the next layer's
// A operand (tiles 0 and 1) or, NARROW, the fp32 dot products of a 3-wide output layer (weights `nw` [3][128]) reduced over
// the four lanes of a row into part[o][row].
template <bool BF16, bool SPLIT, bool RELU, bool BIAS, bool NARROW, int R>
__device__ __forceinline__ void epilogue_wide(unsigned char *a_hi, unsigned char *a_lo, const float (&d)[R], int tid, const float *bias,
                                              const float *nw, float *part) {
    const int lane = tid & 31, wwarp = (tid >> 5) & 3, wg = tid >> 7;
    float dot[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int h = (i >> 1) & 1, row = 64 * wg + frag_row(i, lane, wwarp), col = frag_col(i, lane);
        float x0 = d[i], x1 = d[i + 1];
        if (BIAS) { x0 += bias[col]; x1 += bias[col + 1]; }
        if (RELU) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        if (NARROW) {
#pragma unroll
            for (int o = 0; o < 3; ++o) dot[h][o] = fmaf(x1, nw[o * 128 + col + 1], fmaf(x0, nw[o * 128 + col], dot[h][o]));
        } else {
            store_pair<BF16, SPLIT>(a_hi + (col >> 6) * A_TILE, a_lo + (SPLIT ? (col >> 6) * A_TILE : 0), row, col & 63, x0, x1);
        }
    }
    if (NARROW) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int o = 0; o < 3; ++o) {
                float v = dot[h][o];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                if ((lane & 3) == 0) part[o * TM + 64 * wg + 16 * wwarp + (lane >> 2) + 8 * h] = v;
            }
        }
    }
}

// out of line on purpose (I-cache, register budget of the 2-CTA kernel)
__device__ __noinline__ void lookup8o(const uint4 *lvl, float align_off, bool smoothstep, const uint4 *__restrict__ octs, float u, float v,
                                      float w, float (&f)[16]) {
    lookup8<OCT_F16>(lvl, align_off, smoothstep, octs, u, v, w, f);
}

// Four consecutive levels of a grid -> 8 features (one 16-byte operand chunk): the fp32 quad layout (bf16x3 / bf16 modes) or
// the reference layout.  Out of line on purpose (I-cache).
__device__ __noinline__ void lookup4(const GridMeta &gm, const float2 *__restrict__ table, const float4 *__restrict__ quads, int l0,
                                     float u, float v, float w, float (&f)[8]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 g2 = (gm.dim == 3) ? (quads ? grid_lookup3q(gm, quads, l0 + j, u, v, w) : grid_lookup3(gm, table, l0 + j, u, v, w))
                                        : grid_lookup2(gm, table, l0 + j, u, v);
        f[2 * j] = g2.x;
        f[2 * j + 1] = g2.y;
    }
}

}  // namespace

template <bool BF16, bool SPLIT>
__global__ void __launch_bounds__(HEAD_NT, SPLIT ? 1 : 2) k_head_tc(const __grid_constant__ HeadArgs a, const __grid_constant__ HeadTcArgs t) {
    extern __shared__ __align__(1024) unsigned char smem_raw_[];
    unsigned char *smem_raw = smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u);
    SmemTC<SPLIT> &s = *reinterpret_cast<SmemTC<SPLIT> *>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, wg = tid >> 7, lane = tid & 31;

    // ---- one-time setup ----
    MarchConst mc = a.mc;
    float occ_lo[3] = {0.f, 0.f, 0.f}, occ_hi[3] = {0.f, 0.f, 0.f};
    const bool have_box = setup_occupancy(a, mc, occ_lo, occ_hi);
    install_coarse(a, s, mc, tid, NT);
    if (tid == 32) {
        for (int i = 0; i < W_NSTAGE; ++i) mbar_init(&s.bar_full[i], 1);
        mbar_fence_init();
        s.next = 0; s.end = 0; s.done = 0;
    }
    for (int i = tid; i < 3 * 128; i += NT) {   // a.narrow rows: 0-2 ambient out, 3 sigma, 4-6 color out, 7 color-L0 bias
        s.nw[i] = a.narrow[i];
        s.nw[3 * 128 + i] = a.narrow[4 * 128 + i];
    }
    if (tid < 128) s.bias[tid] = a.narrow[7 * 128 + tid];
    stage_level_meta(a.pos_gm, nullptr, s.lvl[0], tid);
    stage_level_meta(a.amb_gm, nullptr, s.lvl[1], tid);
    fence_async_smem();
    __syncthreads();
    if (warp == 0) {
        if (elect_one()) issue_loads<SPLIT, 0, W_NSTAGE>(t, s);
        __syncwarp();
    }

    const int total = (a.pass == 1) ? *a.n_hits : *a.n_survivors;
    Slot sl;
    sl.active = false;
    sl.gid = 0; sl.frame = 0; sl.nsamp = 0; sl.cap = 0;

    long long ph_last = clock64();
#define PH(i)                                                                                   \
    if (a.phase_cycles && tid == 0) {                                                           \
        const long long now_ = clock64();                                                       \
        atomicAdd(a.phase_cycles + (i), (unsigned long long)(now_ - ph_last));                  \
        ph_last = now_;                                                                         \
    }
    for (;;) {
        // ================= refill dead slots from the global cursor, publish the batch (head_common.cuh) =================
        const int n_valid = refill_and_publish(a, s, sl, mc, have_box, occ_lo, occ_hi, total, tid);
        if (n_valid < 0) break;
        if (n_valid == 0) continue;
        PH(0)   // refill + publish

        const int slot = tid & (TM - 1), lg = tid >> 7;
        const bool v = s.valid[slot] != 0;
        uint4 park_h[2], park_l[2];   // this thread's two position-feature operand chunks, parked across the ambient net
        // ---- position grid -> A tile0 k[0,32) and the park; conditioning -> tile0 k[32,64), tile1 k[0,32) ----
        {
            float u = 0.f, vv = 0.f, w = 0.f;
            if (v) {
                const float inv2b = 2.0f * mc.bound;
                u = __fdiv_rn(__fadd_rn(s.sx[slot], mc.bound), inv2b);
                vv = __fdiv_rn(__fadd_rn(s.sy[slot], mc.bound), inv2b);
                w = __fdiv_rn(__fadd_rn(s.sz[slot], mc.bound), inv2b);
            }
            if (a.pos_octs) {   // thread (slot, lg) owns levels lg*8 .. lg*8+7 = operand chunks 2lg, 2lg+1
                float f[16];
                if (v) lookup8o(&s.lvl[0][lg * 16], a.pos_gm.align_off, a.pos_gm.interp == 1, a.pos_octs, u, vv, w, f);
                else {
#pragma unroll
                    for (int i = 0; i < 16; ++i) f[i] = 0.f;
                }
                store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 2 * lg), &f[0]);
                store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 2 * lg + 1), &f[8]);
            } else {
#pragma unroll 1
                for (int c = 0; c < 2; ++c) {
                    float f[8];
                    if (v) lookup4(a.pos_gm, a.pos_tab, a.pos_quads, lg * 8 + c * 4, u, vv, w, f);
                    else {
#pragma unroll
                        for (int i = 0; i < 8; ++i) f[i] = 0.f;
                    }
                    store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 2 * lg + c), f);
                }
            }
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                park_h[c] = *reinterpret_cast<const uint4 *>(s.a_hi[0] + sw128_off(slot, 2 * lg + c));
                if (SPLIT) park_l[c] = *reinterpret_cast<const uint4 *>(s.a_lo[0] + sw128_off(slot, 2 * lg + c));
            }
            // cond values [lg*32, lg*32+32) sit at k = 32 + lg*32 + i: lg 0 -> tile0 chunks 4..7, lg 1 -> tile1 chunks 0..3
            const float4 *cf = reinterpret_cast<const float4 *>(a.cond_feat + (size_t)s.frame[slot] * 64 + lg * 32);
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                float c8[8];
                if (v) {
                    const float4 q0 = __ldg(cf + 2 * j), q1 = __ldg(cf + 2 * j + 1);
                    c8[0] = q0.x; c8[1] = q0.y; c8[2] = q0.z; c8[3] = q0.w; c8[4] = q1.x; c8[5] = q1.y; c8[6] = q1.z; c8[7] = q1.w;
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) c8[i] = 0.f;
                }
                store_chunk<BF16, SPLIT>(s.a_hi[lg], s.a_lo[SPLIT ? lg : 0], sw128_off(slot, (lg == 0 ? 4 : 0) + j), c8);
            }
        }
        fence_async_smem();
        __syncthreads();
        PH(1)   // position gather + cond + park

        // ---- ambient net 96 -> 128 -> 128 -> 3 ----
        {
            float d[64];
            mma_layer<BF16, SPLIT, 0, 2, 128>(t, s, wg, warp, d);
            PH(2)   // MMA issue + wait (ambient L0)
            epilogue_wide<BF16, SPLIT, true, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], d, tid, nullptr, nullptr, nullptr);
        }
        fence_async_smem(); __syncthreads();
        PH(3)   // epilogue (ambient L0) + barrier
        {
            float d[64];
            mma_layer<BF16, SPLIT, 2, 2, 128>(t, s, wg, warp, d);
            PH(4)   // MMA (ambient L1)
            // ambient L1 epilogue fused with the 3-wide ambient output layer (fp32 dot products straight from the accumulators)
            epilogue_wide<BF16, SPLIT, true, false, true>(&s.a_hi[0][0], &s.a_lo[0][0], d, tid, nullptr, s.nw, s.part);
        }
        __syncthreads();
        PH(5)   // epilogue (ambient L1) + dots
        if (tid < TM) {
            s.amb[tid] = tanhf(s.part[0 * TM + tid]);
            s.amb[TM + tid] = tanhf(s.part[1 * TM + tid]);
            s.amb[2 * TM + tid] = tanhf(s.part[2 * TM + tid]);
        }
        __syncthreads();
        PH(6)   // narrow ambient out: MMA + tanh
        // ---- sigma-net input: tile0 k[0,32) <- parked position features, k[32,64) <- ambient grid ----
        {
            float u = 0.f, vv = 0.f, w = 0.f;
            if (v) {   // GridEncoder.forward with bound = 1: (x + 1) / 2
                u = __fdiv_rn(__fadd_rn(s.amb[slot], 1.0f), 2.0f);
                vv = __fdiv_rn(__fadd_rn(s.amb[TM + slot], 1.0f), 2.0f);
                w = __fdiv_rn(__fadd_rn(s.amb[2 * TM + slot], 1.0f), 2.0f);
            }
#pragma unroll
            for (int c = 0; c < 2; ++c) {   // parked position features back into tile 0, k[0,32)
                *reinterpret_cast<uint4 *>(s.a_hi[0] + sw128_off(slot, 2 * lg + c)) = park_h[c];
                if (SPLIT) *reinterpret_cast<uint4 *>(s.a_lo[0] + sw128_off(slot, 2 * lg + c)) = park_l[c];
            }
            if (a.amb_octs) {
                float f[16];
                if (v) lookup8o(&s.lvl[1][lg * 16], a.amb_gm.align_off, a.amb_gm.interp == 1, a.amb_octs, u, vv, w, f);
                else {
#pragma unroll
                    for (int i = 0; i < 16; ++i) f[i] = 0.f;
                }
                store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 4 + 2 * lg), &f[0]);
                store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 4 + 2 * lg + 1), &f[8]);
            } else {
#pragma unroll 1
                for (int c = 0; c < 2; ++c) {
                    float f[8];
                    if (v) lookup4(a.amb_gm, a.amb_tab, a.amb_quads, lg * 8 + c * 4, u, vv, w, f);
                    else {
#pragma unroll
                        for (int i = 0; i < 8; ++i) f[i] = 0.f;
                    }
                    store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 4 + 2 * lg + c), f);
                }
            }
        }
        fence_async_smem(); __syncthreads();
        PH(7)   // ambient gather + unpark

        // ---- sigma net 64 -> 128 -> 128 -> (128 geo + sigma) ----
        {
            float d[64];
            mma_layer<BF16, SPLIT, 4, 1, 128>(t, s, wg, warp, d);
            epilogue_wide<BF16, SPLIT, true, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], d, tid, nullptr, nullptr, nullptr);
        }
        fence_async_smem(); __syncthreads();
        {
            float d[64];
            mma_layer<BF16, SPLIT, 5, 2, 128>(t, s, wg, warp, d);
            epilogue_wide<BF16, SPLIT, true, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], d, tid, nullptr, nullptr, nullptr);
        }
        fence_async_smem(); __syncthreads();
        {
            float d[72];
            mma_layer<BF16, SPLIT, 7, 2, 144>(t, s, wg, warp, d);
            if ((lane & 3) == 0) {   // column 128 = sigma logit (weight row 0 was packed last); sigma = density_scale * exp(h)
                const int r = 64 * wg + 16 * (warp & 3) + (lane >> 2);
                s.sig[r] = a.density_scale * expf(d[64]);
                s.sig[r + 8] = a.density_scale * expf(d[66]);
            }
            epilogue_wide<BF16, SPLIT, false, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], d, tid, nullptr, nullptr, nullptr);   // geo features -> tiles 0,1 (k = 0..127)
        }
        if (tid < TM) {   // SH(dir) -> K16 tile
            float sh[16];
            sh4(sl.g.dx, sl.g.dy, sl.g.dz, sh);
            if (!sl.active) {
#pragma unroll
                for (int i = 0; i < 16; ++i) sh[i] = 0.f;
            }
            store_chunk<BF16, SPLIT>(s.s_hi, s.s_lo, k16_off(tid, 0), &sh[0]);
            store_chunk<BF16, SPLIT>(s.s_hi, s.s_lo, k16_off(tid, 1), &sh[8]);
        }
        fence_async_smem(); __syncthreads();

        PH(8)   // sigma net: 3 MMA layers + 3 epilogues
        // ---- color net (128 geo + 16 SH [+ folded individual code]) -> 128 -> 3 ----
        {
            float d[64];
            mma_layer<BF16, SPLIT, 9, 3, 128>(t, s, wg, warp, d);
            // color L0 epilogue fused with the 3-wide rgb output layer
            epilogue_wide<BF16, SPLIT, true, true, true>(&s.a_hi[0][0], &s.a_lo[0][0], d, tid, s.bias, s.nw + 3 * 128, s.part);
        }
        __syncthreads();
        if (tid < TM) {
            s.rgb[tid] = 1.0f / (1.0f + expf(-s.part[0 * TM + tid]));
            s.rgb[TM + tid] = 1.0f / (1.0f + expf(-s.part[1 * TM + tid]));
            s.rgb[2 * TM + tid] = 1.0f / (1.0f + expf(-s.part[2 * TM + tid]));
        }
        __syncthreads();

        PH(9)   // color net: 2 MMA layers + epilogue + sigmoid
        // ================= composite + advance (head_common.cuh) =================
        composite_and_advance(a, s, sl, mc, tid);
        PH(10)  // composite + march to next sample
        if (a.phase_cycles && tid == 0) atomicAdd(a.phase_cycles + 31, 1ull);   // batches
        // no barrier needed here: the refill starts with one before shared memory is touched again
    }

    // drain the prefetched weight tiles: the bulk copies must land before the CTA exits
    for (uint32_t q = 0; q < W_NSTAGE; ++q) mbar_wait(&s.bar_full[q], 0);   // tiles 0..2 of a batch that never comes
}

static_assert(sizeof(SmemTC<false>) + 1024 <= 113 * 1024, "single-pass kernel must fit twice per SM (228 KB - 2 x 1 KB reserved)");
static_assert(sizeof(SmemTC<true>) + 1024 <= 227 * 1024, "split kernel exceeds the per-CTA shared memory limit");
size_t head_tc_smem_bytes(bool split) { return (split ? sizeof(SmemTC<true>) : sizeof(SmemTC<false>)) + 1024; }

cudaError_t launch_head_tc(const HeadArgs &a, const HeadTcArgs &t, int precision, int total_hint, cudaStream_t st) {
    const bool split = precision == BF16_X3;
    int blocks = sm_count() * (split ? 1 : 2);   // single-pass kernels: two resident CTAs per SM
    if (getenv("GFPP_ONE_CTA")) blocks = sm_count();   // diagnostics: phase timings without the co-resident CTA
    if (total_hint >= 0) {
        const int need = (total_hint + TM - 1) / TM;
        if (need < blocks) blocks = need > 0 ? need : 1;
    }
    const size_t smem = head_tc_smem_bytes(split);
    cudaError_t e;
#define GO(BF, SP)                                                                                             \
    e = cudaFuncSetAttribute(k_head_tc<BF, SP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);       \
    if (e != cudaSuccess) return e;                                                                            \
    e = cudaFuncSetAttribute(k_head_tc<BF, SP>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared); \
    if (e != cudaSuccess) return e;                                                                            \
    if (getenv("GFPP_DEBUG")) {                                                                                \
        int occ = 0;                                                                                           \
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_head_tc<BF, SP>, NT, smem);                      \
        fprintf(stderr, "[gfpp] k_head_tc<%d,%d>: %zu B smem, %d CTA/SM, grid %d\n", (int)BF, (int)SP, smem, occ, blocks); \
    }                                                                                                          \
    k_head_tc<BF, SP><<<blocks, NT, smem, st>>>(a, t);
    if (precision == FP16_X1) { GO(false, false) }
    else if (precision == BF16_X1) { GO(true, false) }
    else if (precision == BF16_X3) { GO(true, true) }
    else return cudaErrorInvalidValue;
#undef GO
    return cudaGetLastError();
}

// Density query in the fp16 mode (DensityArgs: head_kernel.cuh): the field k_head_tc shades -- fp16 "oct" tables, fp16 operands,
// fp32 accumulation, the same tile stream -- up to the sigma net, for 128 points per batch and no marching.  The colour tiles of the
// static 12-tile schedule are waited for and recycled without MMAs, so stage and parity stay compile-time constants.
template <bool GEO>
__global__ void __launch_bounds__(HEAD_NT, 2) k_density_tc(const __grid_constant__ HeadArgs a, const __grid_constant__ HeadTcArgs t,
                                                          const __grid_constant__ DensityArgs d) {
    constexpr bool BF16 = false, SPLIT = false;
    extern __shared__ __align__(1024) unsigned char smem_raw_[];
    unsigned char *smem_raw = smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u);
    SmemTC<SPLIT> &s = *reinterpret_cast<SmemTC<SPLIT> *>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, wg = tid >> 7, lane = tid & 31;
    if (tid == 32) {
        for (int i = 0; i < W_NSTAGE; ++i) mbar_init(&s.bar_full[i], 1);
        mbar_fence_init();
    }
    for (int i = tid; i < 3 * 128; i += NT) s.nw[i] = a.narrow[i];   // ambient out rows 0-2
    stage_level_meta(a.pos_gm, nullptr, s.lvl[0], tid);
    stage_level_meta(a.amb_gm, nullptr, s.lvl[1], tid);
    fence_async_smem();
    __syncthreads();
    if (warp == 0) {
        if (elect_one()) issue_loads<SPLIT, 0, W_NSTAGE>(t, s);
        __syncwarp();
    }
    const uint32_t n_batches = (d.n + TM - 1) / TM;
    const uint32_t H = d.grid_size, H3 = H * H * H;
    const int slot = tid & (TM - 1), lg = tid >> 7;
    for (uint32_t b = blockIdx.x; b < n_batches; b += gridDim.x) {
        if (tid < TM) {
            float q[3];
            const bool v = density_point(d, b * TM + tid, H, H3, q);
            s.valid[tid] = v ? 1 : 0;
            s.sx[tid] = q[0]; s.sy[tid] = q[1]; s.sz[tid] = q[2];
        }
        __syncthreads();
        const bool v = s.valid[slot] != 0;
        uint4 park_h[2];
        // ---- position grid -> A tile0 k[0,32) and the park; conditioning -> tile0 k[32,64), tile1 k[0,32) (as k_head_tc) ----
        {
            float u = 0.f, vv = 0.f, w = 0.f;
            if (v) {
                const float inv2b = 2.0f * d.bound;
                u = __fdiv_rn(__fadd_rn(s.sx[slot], d.bound), inv2b);
                vv = __fdiv_rn(__fadd_rn(s.sy[slot], d.bound), inv2b);
                w = __fdiv_rn(__fadd_rn(s.sz[slot], d.bound), inv2b);
            }
            float f[16];
            if (v) lookup8o(&s.lvl[0][lg * 16], a.pos_gm.align_off, a.pos_gm.interp == 1, a.pos_octs, u, vv, w, f);
            else {
#pragma unroll
                for (int i = 0; i < 16; ++i) f[i] = 0.f;
            }
            store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 2 * lg), &f[0]);
            store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 2 * lg + 1), &f[8]);
#pragma unroll
            for (int c = 0; c < 2; ++c) park_h[c] = *reinterpret_cast<const uint4 *>(s.a_hi[0] + sw128_off(slot, 2 * lg + c));
            const float4 *cf = reinterpret_cast<const float4 *>(d.cond + lg * 32);
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                float c8[8];
                if (v) {
                    const float4 q0 = __ldg(cf + 2 * j), q1 = __ldg(cf + 2 * j + 1);
                    c8[0] = q0.x; c8[1] = q0.y; c8[2] = q0.z; c8[3] = q0.w; c8[4] = q1.x; c8[5] = q1.y; c8[6] = q1.z; c8[7] = q1.w;
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) c8[i] = 0.f;
                }
                store_chunk<BF16, SPLIT>(s.a_hi[lg], s.a_lo[0], sw128_off(slot, (lg == 0 ? 4 : 0) + j), c8);
            }
        }
        fence_async_smem();
        __syncthreads();
        // ---- ambient net 96 -> 128 -> 128 -> 3, tanh ----
        {
            float dd[64];
            mma_layer<BF16, SPLIT, 0, 2, 128>(t, s, wg, warp, dd);
            epilogue_wide<BF16, SPLIT, true, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], dd, tid, nullptr, nullptr, nullptr);
        }
        fence_async_smem(); __syncthreads();
        {
            float dd[64];
            mma_layer<BF16, SPLIT, 2, 2, 128>(t, s, wg, warp, dd);
            epilogue_wide<BF16, SPLIT, true, false, true>(&s.a_hi[0][0], &s.a_lo[0][0], dd, tid, nullptr, s.nw, s.part);
        }
        __syncthreads();
        if (tid < TM) {
            s.amb[tid] = tanhf(s.part[0 * TM + tid]);
            s.amb[TM + tid] = tanhf(s.part[1 * TM + tid]);
            s.amb[2 * TM + tid] = tanhf(s.part[2 * TM + tid]);
        }
        __syncthreads();
        // ---- sigma-net input: parked position features, ambient grid ----
        {
            float u = 0.f, vv = 0.f, w = 0.f;
            if (v) {
                u = __fdiv_rn(__fadd_rn(s.amb[slot], 1.0f), 2.0f);
                vv = __fdiv_rn(__fadd_rn(s.amb[TM + slot], 1.0f), 2.0f);
                w = __fdiv_rn(__fadd_rn(s.amb[2 * TM + slot], 1.0f), 2.0f);
            }
#pragma unroll
            for (int c = 0; c < 2; ++c) *reinterpret_cast<uint4 *>(s.a_hi[0] + sw128_off(slot, 2 * lg + c)) = park_h[c];
            float f[16];
            if (v) lookup8o(&s.lvl[1][lg * 16], a.amb_gm.align_off, a.amb_gm.interp == 1, a.amb_octs, u, vv, w, f);
            else {
#pragma unroll
                for (int i = 0; i < 16; ++i) f[i] = 0.f;
            }
            store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 4 + 2 * lg), &f[0]);
            store_chunk<BF16, SPLIT>(s.a_hi[0], s.a_lo[0], sw128_off(slot, 4 + 2 * lg + 1), &f[8]);
        }
        fence_async_smem(); __syncthreads();
        // ---- sigma net 64 -> 128 -> 128 -> (128 geo + sigma) ----
        {
            float dd[64];
            mma_layer<BF16, SPLIT, 4, 1, 128>(t, s, wg, warp, dd);
            epilogue_wide<BF16, SPLIT, true, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], dd, tid, nullptr, nullptr, nullptr);
        }
        fence_async_smem(); __syncthreads();
        {
            float dd[64];
            mma_layer<BF16, SPLIT, 5, 2, 128>(t, s, wg, warp, dd);
            epilogue_wide<BF16, SPLIT, true, false, false>(&s.a_hi[0][0], &s.a_lo[0][0], dd, tid, nullptr, nullptr, nullptr);
        }
        fence_async_smem(); __syncthreads();
        {
            float dd[72];
            mma_layer<BF16, SPLIT, 7, 2, 144>(t, s, wg, warp, dd);
            const int wwarp = warp & 3;
            if ((lane & 3) == 0) {   // column 128 = sigma logit
                const uint32_t p = b * TM + 64 * wg + 16 * wwarp + (lane >> 2);
                if (p < d.n) d.sigma[p] = __fmul_rn(expf(dd[64]), d.out_scale);
                if (p + 8 < d.n) d.sigma[p + 8] = __fmul_rn(expf(dd[66]), d.out_scale);
            }
            if (GEO) {
#pragma unroll
                for (int i = 0; i < 64; i += 2) {
                    const uint32_t p = b * TM + 64 * wg + frag_row(i, lane, wwarp);
                    if (p < d.n) *reinterpret_cast<float2 *>(d.geo + (size_t)p * 128 + frag_col(i, lane)) = make_float2(dd[i], dd[i + 1]);
                }
            }
        }
        // ---- the colour tiles 9..11 of the static schedule: wait for them and recycle their stages for the next batch ----
#pragma unroll
        for (int c = 9; c < 12; ++c) mbar_wait(&s.bar_full[c % W_NSTAGE], (c / W_NSTAGE) & 1);
        __syncthreads();
        if (warp == 0) {
            if (elect_one()) issue_loads<SPLIT, 12, 3>(t, s);
            __syncwarp();
        }
    }
    for (uint32_t q = 0; q < W_NSTAGE; ++q) mbar_wait(&s.bar_full[q], 0);   // tiles 0..2 of a batch that never comes
}

cudaError_t launch_density_tc(const HeadArgs &a, const HeadTcArgs &t, const DensityArgs &d, cudaStream_t st) {
    if (d.n == 0) return cudaSuccess;
    auto kern = d.geo ? k_density_tc<true> : k_density_tc<false>;
    const size_t smem = head_tc_smem_bytes(false);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    const uint32_t need = (d.n + TM - 1) / TM, cap = 2u * (uint32_t)sm_count();
    kern<<<need < cap ? need : cap, NT, smem, st>>>(a, t, d);
    return cudaGetLastError();
}

}  // namespace gfpp
