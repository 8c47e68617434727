// head_kernel.cu -- fused persistent head renderer (fp32 FFMA variant).
//
// Replaces the host-driven loop of NeRFRenderer.render (modules/radnerfs/renderer.py:340-384):
//   near_far_from_aabb -> [march_rays -> GridEncoder -> ambient MLP -> GridEncoder -> sigma MLP ->
//   SHEncoder -> color MLP -> composite_rays -> compaction]* ,  ~40 launches + 1 host sync per round,
// with ONE persistent kernel per pass.  No intermediate (xyzs/dirs/deltas/features/activations) ever
// leaves the SM.
//
// Shape of the computation
//   * one CTA per SM, 256 threads, a pool of TM=128 ray slots; a slot is owned by thread `slot` (<128)
//     which keeps the ray state (origin, dir, t, accumulators) in registers for the ray's lifetime;
//   * every round each live slot contributes its next occupied sample -> a 128-row batch;
//     dead slots are refilled from a global work cursor (persistent threads with ray refill), so batches
//     stay full regardless of where rays terminate; rays of different frames may share a batch
//     (the per-frame conditioning vector is part of the A tile, exactly as in the reference: K=96);
//   * the batch runs the three MLPs as 128x128xK fp32 FFMA tile GEMMs out of shared memory; weights
//     are streamed layer-chunk by layer-chunk through a 2-stage ring with cp.async.bulk (TMA bulk copy)
//     + mbarrier, prefetching across layer and batch boundaries;
//   * hash-grid features are gathered straight into the A tile (tables are L2-resident: 14.4 MB);
//   * compositing is sequential per ray in the owner thread -> same order as the reference.
//
// Round-schedule exactness (SURVEY.md H1): the reference stops a ray after B = sum_j n_step_j samples where
// n_step_j depends on the global alive count.  Pass 1 renders every ray up to max_steps samples and
// histograms the death index D of each ray; k_schedule replays the n_step recurrence on the histogram
// (it only needs counts of D < max_steps, which pass 1 knows exactly) to get B; pass 2 resumes the rays
// that outlived max_steps for B - max_steps more samples.  No host synchronisation anywhere.
#include "common.cuh"
#include "head_common.cuh"
#include "head_kernel.cuh"
#include "launch.cuh"

namespace gfpp {

namespace {

constexpr int TM = HEAD_TM;
constexpr int NT = HEAD_NT;
constexpr int LDA = 148;                  // A-tile row stride in floats (16B aligned, 148 % 32 = 20)
constexpr int LDP = 36;                   // position-feature copy stride
constexpr int WCHUNK = 72 * 128;          // floats per weight stage (largest chunk: 72 k-rows)
constexpr int NSTAGE = 2;

struct Smem {
    float A[TM * LDA];
    float P[TM * LDP];
    float W[NSTAGE * WCHUNK];
    float narrow[8 * 128];   // rows: amb2[0..2], sigma row, col1[0..2], color-L0 bias (individual code folded)
    float sx[TM], sy[TM], sz[TM];
    float amb[3 * TM];
    float sig[TM];
    float rgb[3 * TM];
    int frame[TM];
    int valid[TM];
    unsigned long long bar[NSTAGE];
    uint32_t coarse[HEAD_COARSE_WORDS];
    int next, end, done;
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Weight-stream state: chunk ids cycle 0..HEAD_NCHUNK-1 forever; `consumed` is uniform across the CTA.
struct WStream {
    uint32_t consumed;
};

// NC: chunks per batch -- the stream cycles through chunks 0..NC-1 (k_density stops before the colour net's chunks)
template <int NC = HEAD_NCHUNK>
__device__ __forceinline__ void issue_chunk(const HeadArgs &a, Smem &s, uint32_t seq) {
    const uint32_t stage = seq % NSTAGE, id = seq % NC;
    const uint32_t bytes = (uint32_t)a.chunk_k[id] * 128u * 4u;
    mbar_expect_tx(&s.bar[stage], bytes);
    bulk_g2s(s.W + stage * WCHUNK, a.wide + a.chunk_off[id], bytes, &s.bar[stage]);
}

// acc[i][j] += A[row_i][kbase + k] * W[k][col_j] for k in [0, kc).   rows: ty*4+i (i<4), 64+ty*4+(i-4);
// cols: tx*4+j (j<4), 64+tx*4+(j-4).  A is row-major (stride LDA), W is k-major [kc][128].
__device__ __forceinline__ void ffma_chunk(float (&acc)[8][8], const float *__restrict__ sA, const float *__restrict__ sW,
                                           int kbase, int kc, int ty, int tx) {
    const float *a0 = sA + (ty * 4) * LDA + kbase;
    const float *a1 = sA + (64 + ty * 4) * LDA + kbase;
    const float *w = sW + tx * 4;
#pragma unroll 2
    for (int k4 = 0; k4 < kc; k4 += 4) {
        float4 av[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            av[i] = *reinterpret_cast<const float4 *>(a0 + i * LDA + k4);
            av[4 + i] = *reinterpret_cast<const float4 *>(a1 + i * LDA + k4);
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const float4 b0 = *reinterpret_cast<const float4 *>(w + (k4 + kk) * 128);
            const float4 b1 = *reinterpret_cast<const float4 *>(w + (k4 + kk) * 128 + 64);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float ai = kk == 0 ? av[i].x : kk == 1 ? av[i].y : kk == 2 ? av[i].z : av[i].w;
                acc[i][0] = fmaf(ai, b0.x, acc[i][0]);
                acc[i][1] = fmaf(ai, b0.y, acc[i][1]);
                acc[i][2] = fmaf(ai, b0.z, acc[i][2]);
                acc[i][3] = fmaf(ai, b0.w, acc[i][3]);
                acc[i][4] = fmaf(ai, b1.x, acc[i][4]);
                acc[i][5] = fmaf(ai, b1.y, acc[i][5]);
                acc[i][6] = fmaf(ai, b1.z, acc[i][6]);
                acc[i][7] = fmaf(ai, b1.w, acc[i][7]);
            }
        }
    }
}

// One 128x128xK layer: consume `nchunks` chunks from the stream, then write act(acc + bias) to A[:, coff:coff+128].
template <bool RELU, int NC = HEAD_NCHUNK>
__device__ __forceinline__ void wide_layer(const HeadArgs &a, Smem &s, WStream &ws, int nchunks, int coff,
                                           const float *bias, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    int kbase = 0;
    for (int c = 0; c < nchunks; ++c) {
        const uint32_t seq = ws.consumed, stage = seq % NSTAGE, id = seq % NC;
        const int kc = a.chunk_k[id];
        mbar_wait(&s.bar[stage], (seq / NSTAGE) & 1);
        ffma_chunk(acc, s.A, s.W + stage * WCHUNK, kbase, kc, ty, tx);
        kbase += kc;
        ws.consumed = seq + 1;
        __syncthreads();  // everyone is done with this stage (and, after the last chunk, with reading A)
        if (tid == 0) issue_chunk<NC>(a, s, seq + NSTAGE);
    }
    float bv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bv[j] = bias ? bias[(j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4))] : 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4);
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            v[j] = acc[i][j] + bv[j];
            if (RELU) v[j] = fmaxf(v[j], 0.f);
        }
        float *dst = s.A + row * LDA + coff + tx * 4;
        *reinterpret_cast<float4 *>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4 *>(dst + 64) = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncthreads();
}

// dot products of every row of A[:, 0:128] with NOUT narrow weight rows; both lanes of a pair get the sums.
template <int NOUT>
__device__ __forceinline__ void narrow_dot(const Smem &s, const float *wrow, int tid, float (&out)[NOUT]) {
    const int row = tid >> 1, half = tid & 1;
    const float *ar = s.A + row * LDA + half * 64;
    float v[NOUT];
#pragma unroll
    for (int o = 0; o < NOUT; ++o) v[o] = 0.f;
#pragma unroll 4
    for (int k = 0; k < 64; k += 4) {
        const float4 x = *reinterpret_cast<const float4 *>(ar + k);
#pragma unroll
        for (int o = 0; o < NOUT; ++o) {
            const float4 w = *reinterpret_cast<const float4 *>(wrow + o * 128 + half * 64 + k);
            v[o] = fmaf(x.x, w.x, v[o]);
            v[o] = fmaf(x.y, w.y, v[o]);
            v[o] = fmaf(x.z, w.z, v[o]);
            v[o] = fmaf(x.w, w.w, v[o]);
        }
    }
#pragma unroll
    for (int o = 0; o < NOUT; ++o) out[o] = v[o] + __shfl_xor_sync(0xffffffffu, v[o], 1);
}

using namespace headc;

}  // namespace

__global__ void __launch_bounds__(HEAD_NT, 1) k_head(const __grid_constant__ HeadArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x;

    // ---- one-time setup ----
    MarchConst mc = a.mc;
    float occ_lo[3] = {0.f, 0.f, 0.f}, occ_hi[3] = {0.f, 0.f, 0.f};
    const bool have_box = setup_occupancy(a, mc, occ_lo, occ_hi);
    install_coarse(a, s, mc, tid, NT);
    for (int i = tid; i < 8 * 128; i += NT) s.narrow[i] = a.narrow[i];
    if (tid == 0) {
        for (int i = 0; i < NSTAGE; ++i) mbar_init(&s.bar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        s.next = 0; s.end = 0; s.done = 0;
    }
    __syncthreads();
    if (tid == 0)
        for (uint32_t q = 0; q < NSTAGE; ++q) issue_chunk(a, s, q);
    WStream wst;
    wst.consumed = 0;

    const int total = (a.pass == 1) ? *a.n_hits : *a.n_survivors;
    Slot sl;
    sl.active = false;
    sl.gid = 0; sl.frame = 0; sl.nsamp = 0; sl.cap = 0;

    for (;;) {
        // ================= refill dead slots from the global cursor, publish the batch (head_common.cuh) =================
        const int n_valid = refill_and_publish(a, s, sl, mc, have_box, occ_lo, occ_hi, total, tid);
        if (n_valid < 0) break;
        if (n_valid == 0) continue;

        const int slot = tid & (TM - 1), lg = tid >> 7;
        const bool v = s.valid[slot] != 0;
        // ---- position grid -> A[:, 0:32] (+ copy in P); conditioning -> A[:, 32:96] ----
        {
            float *ar = s.A + slot * LDA, *pr = s.P + slot * LDP;
            if (v) {
                const float inv2b = 2.0f * mc.bound;
                const float u = __fdiv_rn(__fadd_rn(s.sx[slot], mc.bound), inv2b);
                const float vv = __fdiv_rn(__fadd_rn(s.sy[slot], mc.bound), inv2b);
                const float w = __fdiv_rn(__fadd_rn(s.sz[slot], mc.bound), inv2b);
#pragma unroll 2
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    const float2 f = a.pos_quads ? grid_lookup3q(a.pos_gm, a.pos_quads, l, u, vv, w) : grid_lookup3(a.pos_gm, a.pos_tab, l, u, vv, w);
                    *reinterpret_cast<float2 *>(ar + 2 * l) = f;
                    *reinterpret_cast<float2 *>(pr + 2 * l) = f;
                }
                const float4 *cf = reinterpret_cast<const float4 *>(a.cond_feat + (size_t)s.frame[slot] * 64 + lg * 32);
#pragma unroll
                for (int j = 0; j < 8; ++j) *reinterpret_cast<float4 *>(ar + 32 + lg * 32 + 4 * j) = __ldg(cf + j);
            } else {
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    *reinterpret_cast<float2 *>(ar + 2 * l) = make_float2(0.f, 0.f);
                    *reinterpret_cast<float2 *>(pr + 2 * l) = make_float2(0.f, 0.f);
                }
                for (int j = 0; j < 8; ++j)
                    *reinterpret_cast<float4 *>(ar + 32 + lg * 32 + 4 * j) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        __syncthreads();

        // ---- ambient net 96 -> 128 -> 128 -> 3, tanh (radnerf.py:120-122) ----
        wide_layer<true>(a, s, wst, 2, 0, nullptr, tid);
        wide_layer<true>(a, s, wst, 2, 0, nullptr, tid);
        {
            float o[3];
            narrow_dot<3>(s, s.narrow, tid, o);
            if ((tid & 1) == 0) {
                const int row = tid >> 1;
                s.amb[row] = tanhf(o[0]);
                s.amb[TM + row] = tanhf(o[1]);
                s.amb[2 * TM + row] = tanhf(o[2]);
            }
        }
        __syncthreads();
        // ---- ambient grid -> A[:, 32:64]; A[:, 0:32] <- position features (radnerf.py:123-126) ----
        {
            float *ar = s.A + slot * LDA;
            const float *pr = s.P + slot * LDP;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                *reinterpret_cast<float4 *>(ar + lg * 16 + 4 * j) = *reinterpret_cast<const float4 *>(pr + lg * 16 + 4 * j);
            if (v) {
                // GridEncoder.forward with bound=1: (x + 1) / 2
                const float u = __fdiv_rn(__fadd_rn(s.amb[slot], 1.0f), 2.0f);
                const float vv = __fdiv_rn(__fadd_rn(s.amb[TM + slot], 1.0f), 2.0f);
                const float w = __fdiv_rn(__fadd_rn(s.amb[2 * TM + slot], 1.0f), 2.0f);
#pragma unroll 2
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    const float2 f = (a.amb_gm.dim == 3) ? (a.amb_quads ? grid_lookup3q(a.amb_gm, a.amb_quads, l, u, vv, w) : grid_lookup3(a.amb_gm, a.amb_tab, l, u, vv, w))
                                                         : grid_lookup2(a.amb_gm, a.amb_tab, l, u, vv);
                    *reinterpret_cast<float2 *>(ar + 32 + 2 * l) = f;
                }
            } else {
                for (int l = lg * 8; l < lg * 8 + 8; ++l) *reinterpret_cast<float2 *>(ar + 32 + 2 * l) = make_float2(0.f, 0.f);
            }
        }
        __syncthreads();

        // ---- sigma net 64 -> 128 -> 128 -> (1 + 128) (radnerf.py:126-130) ----
        wide_layer<true>(a, s, wst, 1, 0, nullptr, tid);
        wide_layer<true>(a, s, wst, 2, 0, nullptr, tid);
        {
            float o[1];
            narrow_dot<1>(s, s.narrow + 3 * 128, tid, o);
            // trunc_exp forward is plain exp (utils.py:36-41); sigmas *= density_scale (renderer.py:376)
            if ((tid & 1) == 0) s.sig[tid >> 1] = a.density_scale * expf(o[0]);
        }
        // geo features (no activation) -> A[:, 16:144]; the k-loop only reads A, the write happens after its
        // trailing barrier, so the sigma dot above needs no extra sync.
        {
            const int ty = tid >> 4, tx = tid & 15;
            float acc[8][8];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
            int kbase = 0;
            for (int c = 0; c < 2; ++c) {
                const uint32_t seq = wst.consumed, stage = seq % NSTAGE, id = seq % HEAD_NCHUNK;
                const int kc = a.chunk_k[id];
                mbar_wait(&s.bar[stage], (seq / NSTAGE) & 1);
                ffma_chunk(acc, s.A, s.W + stage * WCHUNK, kbase, kc, ty, tx);
                kbase += kc;
                wst.consumed = seq + 1;
                __syncthreads();
                if (tid == 0) issue_chunk(a, s, seq + NSTAGE);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int row = i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4);
                float *dst = s.A + row * LDA + 16 + tx * 4;
                *reinterpret_cast<float4 *>(dst) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
                *reinterpret_cast<float4 *>(dst + 64) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
            }
            if (tid < TM) {  // SH(dir) -> A[:, 0:16] (radnerf.py:132-134)
                float sh[16];
                sh4(sl.g.dx, sl.g.dy, sl.g.dz, sh);
                float *dst = s.A + tid * LDA;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    *reinterpret_cast<float4 *>(dst + 4 * j) = sl.active ? make_float4(sh[4 * j], sh[4 * j + 1], sh[4 * j + 2], sh[4 * j + 3])
                                                                         : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            __syncthreads();
        }

        // ---- color net (16 + 128 [+ 4 folded into the bias]) -> 128 -> 3, sigmoid (radnerf.py:134-139) ----
        wide_layer<true>(a, s, wst, 2, 0, s.narrow + 7 * 128, tid);
        {
            float o[3];
            narrow_dot<3>(s, s.narrow + 4 * 128, tid, o);
            if ((tid & 1) == 0) {
                const int row = tid >> 1;
                s.rgb[row] = 1.0f / (1.0f + expf(-o[0]));
                s.rgb[TM + row] = 1.0f / (1.0f + expf(-o[1]));
                s.rgb[2 * TM + row] = 1.0f / (1.0f + expf(-o[2]));
            }
        }
        __syncthreads();

        // ================= composite + advance (head_common.cuh) =================
        composite_and_advance(a, s, sl, mc, tid);
        // no barrier needed here: the refill starts with one before shared memory is touched again
    }

    // drain the prefetched weight chunks before the CTA (and its shared memory) goes away
    for (uint32_t q = 0; q < NSTAGE; ++q) {
        const uint32_t seq = wst.consumed + q;
        mbar_wait(&s.bar[seq % NSTAGE], (seq / NSTAGE) & 1);
    }
}

// Density query (radnerf.py:143-166): position grid -> ambient net -> tanh -> ambient grid -> sigma net, 128 points per batch,
// the same shared-memory FFMA tile GEMMs and weight stream as k_head, but the stream stops after the sigma net (7 chunks, or 9
// when the 128 geo columns of its last layer are wanted).  Persistent CTAs take batches round-robin; nothing is marched.
// In cell mode a batch is 128 consecutive Morton codes, i.e. a 4x4x8 brick, so a warp's corner gathers share sectors.
template <bool GEO>
__global__ void __launch_bounds__(HEAD_NT, 1) k_density(const __grid_constant__ HeadArgs a, const __grid_constant__ DensityArgs d) {
    constexpr int NC = GEO ? 9 : 7;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x;
    for (int i = tid; i < 4 * 128; i += NT) s.narrow[i] = a.narrow[i];   // ambient out rows 0-2, sigma row
    if (tid == 0) {
        for (int i = 0; i < NSTAGE; ++i) mbar_init(&s.bar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
        for (uint32_t q = 0; q < NSTAGE; ++q) issue_chunk<NC>(a, s, q);
    WStream wst;
    wst.consumed = 0;

    const uint32_t n_batches = (d.n + TM - 1) / TM;
    const uint32_t H = d.grid_size, H3 = H * H * H;
    const int slot = tid & (TM - 1), lg = tid >> 7;
    for (uint32_t b = blockIdx.x; b < n_batches; b += gridDim.x) {
        if (tid < TM) {
            float q[3];
            const bool v = density_point(d, b * TM + tid, H, H3, q);
            const float x = q[0], y = q[1], z = q[2];
            s.valid[tid] = v ? 1 : 0;
            s.sx[tid] = x; s.sy[tid] = y; s.sz[tid] = z;
        }
        __syncthreads();
        const bool v = s.valid[slot] != 0;
        // ---- position grid -> A[:, 0:32] (+ copy in P); conditioning -> A[:, 32:96] (as k_head) ----
        {
            float *ar = s.A + slot * LDA, *pr = s.P + slot * LDP;
            if (v) {
                const float inv2b = 2.0f * d.bound;
                const float u = __fdiv_rn(__fadd_rn(s.sx[slot], d.bound), inv2b);
                const float vv = __fdiv_rn(__fadd_rn(s.sy[slot], d.bound), inv2b);
                const float w = __fdiv_rn(__fadd_rn(s.sz[slot], d.bound), inv2b);
#pragma unroll 2
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    const float2 f = a.pos_quads ? grid_lookup3q(a.pos_gm, a.pos_quads, l, u, vv, w) : grid_lookup3(a.pos_gm, a.pos_tab, l, u, vv, w);
                    *reinterpret_cast<float2 *>(ar + 2 * l) = f;
                    *reinterpret_cast<float2 *>(pr + 2 * l) = f;
                }
            } else {
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    *reinterpret_cast<float2 *>(ar + 2 * l) = make_float2(0.f, 0.f);
                    *reinterpret_cast<float2 *>(pr + 2 * l) = make_float2(0.f, 0.f);
                }
            }
            const float4 *cf = reinterpret_cast<const float4 *>(d.cond + lg * 32);
#pragma unroll
            for (int j = 0; j < 8; ++j) *reinterpret_cast<float4 *>(ar + 32 + lg * 32 + 4 * j) = __ldg(cf + j);
        }
        __syncthreads();

        // ---- ambient net 96 -> 128 -> 128 -> 3, tanh ----
        wide_layer<true, NC>(a, s, wst, 2, 0, nullptr, tid);
        wide_layer<true, NC>(a, s, wst, 2, 0, nullptr, tid);
        {
            float o[3];
            narrow_dot<3>(s, s.narrow, tid, o);
            if ((tid & 1) == 0) {
                const int row = tid >> 1;
                s.amb[row] = tanhf(o[0]);
                s.amb[TM + row] = tanhf(o[1]);
                s.amb[2 * TM + row] = tanhf(o[2]);
            }
        }
        __syncthreads();
        // ---- ambient grid -> A[:, 32:64]; A[:, 0:32] <- position features ----
        {
            float *ar = s.A + slot * LDA;
            const float *pr = s.P + slot * LDP;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                *reinterpret_cast<float4 *>(ar + lg * 16 + 4 * j) = *reinterpret_cast<const float4 *>(pr + lg * 16 + 4 * j);
            if (v) {
                const float u = __fdiv_rn(__fadd_rn(s.amb[slot], 1.0f), 2.0f);
                const float vv = __fdiv_rn(__fadd_rn(s.amb[TM + slot], 1.0f), 2.0f);
                const float w = __fdiv_rn(__fadd_rn(s.amb[2 * TM + slot], 1.0f), 2.0f);
#pragma unroll 2
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    const float2 f = (a.amb_gm.dim == 3) ? (a.amb_quads ? grid_lookup3q(a.amb_gm, a.amb_quads, l, u, vv, w) : grid_lookup3(a.amb_gm, a.amb_tab, l, u, vv, w))
                                                         : grid_lookup2(a.amb_gm, a.amb_tab, l, u, vv);
                    *reinterpret_cast<float2 *>(ar + 32 + 2 * l) = f;
                }
            } else {
                for (int l = lg * 8; l < lg * 8 + 8; ++l) *reinterpret_cast<float2 *>(ar + 32 + 2 * l) = make_float2(0.f, 0.f);
            }
        }
        __syncthreads();

        // ---- sigma net 64 -> 128 -> 128 -> (1 + 128) ----
        wide_layer<true, NC>(a, s, wst, 1, 0, nullptr, tid);
        wide_layer<true, NC>(a, s, wst, 2, 0, nullptr, tid);
        {
            float o[1];
            narrow_dot<1>(s, s.narrow + 3 * 128, tid, o);
            const uint32_t p = b * TM + (tid >> 1);
            // trunc_exp forward is plain exp (utils.py:36-41)
            if ((tid & 1) == 0 && p < d.n) d.sigma[p] = __fmul_rn(expf(o[0]), d.out_scale);
        }
        if (GEO) {   // geo features h[1:129], no activation, straight from the accumulators
            const int ty = tid >> 4, tx = tid & 15;
            float acc[8][8];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
            int kbase = 0;
            for (int c = 0; c < 2; ++c) {
                const uint32_t seq = wst.consumed, stage = seq % NSTAGE, id = seq % NC;
                const int kc = a.chunk_k[id];
                mbar_wait(&s.bar[stage], (seq / NSTAGE) & 1);
                ffma_chunk(acc, s.A, s.W + stage * WCHUNK, kbase, kc, ty, tx);
                kbase += kc;
                wst.consumed = seq + 1;
                __syncthreads();
                if (tid == 0) issue_chunk<NC>(a, s, seq + NSTAGE);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int row = i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4);
                const uint32_t p = b * TM + row;
                if (p < d.n) {
                    float *dst = d.geo + (size_t)p * 128 + tx * 4;
                    *reinterpret_cast<float4 *>(dst) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
                    *reinterpret_cast<float4 *>(dst + 64) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
                }
            }
        }
        __syncthreads();   // A, P and the batch's positions are rewritten by the next batch
    }
    for (uint32_t q = 0; q < NSTAGE; ++q) {
        const uint32_t seq = wst.consumed + q;
        mbar_wait(&s.bar[seq % NSTAGE], (seq / NSTAGE) & 1);
    }
}

cudaError_t launch_density(const HeadArgs &a, const DensityArgs &d, cudaStream_t st) {
    if (d.n == 0) return cudaSuccess;
    auto kern = d.geo ? k_density<true> : k_density<false>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    const uint32_t need = (d.n + TM - 1) / TM;
    const int blocks = (int)(need < (uint32_t)sm_count() ? need : (uint32_t)sm_count());
    kern<<<blocks, NT, sizeof(Smem), st>>>(a, d);
    return cudaGetLastError();
}

// Ray setup: one thread per (frame, ray).  Generates / loads the ray, slab-tests it, and marches it to its FIRST occupied
// sample with full occupancy (64 warps/SM hide the dependent bitfield reads).  Rays without any sample (57 % of a
// talking-head frame) are finished here: zero colour/alpha, normalised depth, death index 1.  The others are appended to
// the hit list {ray id, t_pre}; the persistent head kernel adopts them in O(1), so no first-hit marching ever sits
// between two CTA barriers of the MLP pipeline.
__global__ void __launch_bounds__(256) k_ray_setup(const __grid_constant__ HeadArgs a) {
    MarchConst mc = a.mc;
    float occ_lo[3] = {0.f, 0.f, 0.f}, occ_hi[3] = {0.f, 0.f, 0.f};
    const bool have_box = setup_occupancy(a, mc, occ_lo, occ_hi);
    mc.coarse = a.coarse_bits;
    const int total = a.n_frames * a.n_rays;
    for (int gid = blockIdx.x * blockDim.x + threadIdx.x; gid < total; gid += gridDim.x * blockDim.x) {
        Slot sl;
        sl.gid = gid;
        sl.frame = gid / a.n_rays;
        load_ray(a, sl.frame, gid - sl.frame * a.n_rays, sl.g);
        near_far(sl.g, a.aabb, a.min_near, sl.near, sl.far);
        sl.t = sl.near;
        int budget = 1 << 30;
        const bool hit = may_hit_occupied(have_box, occ_lo, occ_hi, sl.g, sl.near, sl.far, sl.far_m) &&
                         march_budget(mc, sl.g, sl.far_m, sl.t, budget) == 1;
        if (hit) {
            cg::coalesced_group grp = cg::coalesced_threads();
            int base = 0;
            if (grp.thread_rank() == 0) base = atomicAdd(a.n_hits, (int)grp.size());
            base = grp.shfl(base, 0);
            HitRecord hr;
            hr.gid = gid; hr.pad = 0;
            sample_at(mc, sl.g, sl.t, hr.t, hr.px, hr.py, hr.pz, hr.dt);
            hr.near = sl.near; hr.far = sl.far; hr.far_m = sl.far_m;
            hr.ox = sl.g.ox; hr.oy = sl.g.oy; hr.oz = sl.g.oz; hr.dx = sl.g.dx; hr.dy = sl.g.dy; hr.dz = sl.g.dz;
            uint4 *dst = a.hits + 4 * (size_t)(base + grp.thread_rank());
            const uint4 *src = reinterpret_cast<const uint4 *>(&hr);
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[i] = src[i];
        } else {
            sl.ws = 0.f; sl.depth = 0.f; sl.r = sl.gch = sl.b = 0.f;
            finalize_ray(a, sl, true);
            warp_agg_add(a.hist, sl.frame * (a.max_steps + 2) + 1, 1);
        }
    }
}

// Replays the reference's round schedule (renderer.py:354-384) on the death histogram of each frame:
//   n_step_j = clamp(N // n_alive_j, 1, 8);  cum += n_step_j;  n_alive_{j+1} = #{D > cum};  until cum >= max_steps.
__global__ void k_schedule(const int *__restrict__ hist, int n_frames, int n_rays, int max_steps, int *__restrict__ B_total) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const int *h = hist + (size_t)f * (max_steps + 2);
    int cum = 0, alive = n_rays, dead_upto = 0, scanned = 0;
    while (cum < max_steps && alive > 0) {
        int n_step = n_rays / alive;
        n_step = n_step < 1 ? 1 : (n_step > 8 ? 8 : n_step);
        cum += n_step;
        const int lim = cum < max_steps + 1 ? cum : max_steps + 1;
        while (scanned < lim) { ++scanned; dead_upto += h[scanned]; }
        alive = n_rays - dead_upto;
    }
    B_total[f] = cum;
}

// debug: the rays the fused path generates in-kernel (load_ray, head_common.cuh) written out like get_rays would (utils.py:352-360)
__global__ void k_dump_rays(const __grid_constant__ HeadArgs a, float *__restrict__ rays_o, float *__restrict__ rays_d) {
    const int total = a.n_frames * a.n_rays;
    for (int gid = blockIdx.x * blockDim.x + threadIdx.x; gid < total; gid += gridDim.x * blockDim.x) {
        const int f = gid / a.n_rays;
        RayGeom g;
        load_ray(a, f, gid - f * a.n_rays, g);
        rays_o[3 * (size_t)gid] = g.ox; rays_o[3 * (size_t)gid + 1] = g.oy; rays_o[3 * (size_t)gid + 2] = g.oz;
        rays_d[3 * (size_t)gid] = g.dx; rays_d[3 * (size_t)gid + 1] = g.dy; rays_d[3 * (size_t)gid + 2] = g.dz;
    }
}
cudaError_t launch_dump_rays(const HeadArgs &a, float *rays_o, float *rays_d, cudaStream_t st) {
    k_dump_rays<<<grid_for((uint64_t)a.n_frames * a.n_rays, 256), 256, 0, st>>>(a, rays_o, rays_d);
    return cudaGetLastError();
}

size_t head_smem_bytes() { return sizeof(Smem); }

cudaError_t launch_head(const HeadArgs &a, int total_hint, cudaStream_t st) {
    // function attributes are per device: set on every launch, never cached process-wide
    cudaError_t e = cudaFuncSetAttribute(k_head, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    int blocks = sm_count();
    if (total_hint >= 0) {
        const int need = (total_hint + TM - 1) / TM;
        if (need < blocks) blocks = need > 0 ? need : 1;
    }
    k_head<<<blocks, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_ray_setup(const HeadArgs &a, cudaStream_t st) {
    const uint64_t total = (uint64_t)a.n_frames * a.n_rays;
    k_ray_setup<<<grid_for(total, 256), 256, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_schedule(const int *hist, int n_frames, int n_rays, int max_steps, int *B_total, cudaStream_t st) {
    k_schedule<<<(n_frames + 63) / 64, 64, 0, st>>>(hist, n_frames, n_rays, max_steps, B_total);
    return cudaGetLastError();
}

}  // namespace gfpp
