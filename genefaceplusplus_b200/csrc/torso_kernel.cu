// torso_kernel.cu -- torso field + final composite (the epilogue of every frame).
//
// Replaces radnerf_torso.py:156-197 (mask by grid_sample of density_grid_torso, forward_torso on the
// masked pixels :51-84, three-way composite, clamp) and, for the head-only model, renderer.py:386-392.
// One persistent kernel: a CTA takes tiles of 128 consecutive pixels of one frame; tiles with no torso
// pixel skip the MLPs.  Per-frame constants (freq-encoded pose, torso code) are folded into per-frame
// bias vectors by k_torso_frame_bias, so the per-pixel GEMMs only see the pixel-dependent columns
// (deform: 42 of 104, canonical: 74 of 136).
//
// The four wide layers (deform 48->64->64, canonical 80->32->32) run on the tensor cores in split tf32 in every precision
// mode: x = hi + lo with hi = rna_tf32(x), lo = rna_tf32(x - hi) (~21-22 bits at every magnitude: tf32 keeps fp32's
// exponent), D = A_lo W_hi + A_hi W_lo + A_hi W_hi with fp32 accumulation (tc.cuh, wgmma_tf32x3).  Warpgroup g owns the
// tile's rows 64g..64g+63 (M = 64); the weights' tf32 hi / lo images (84 KB, torso_kernel.cuh) stay resident in shared
// memory, filled once by one bulk copy.  The A operand comes from REGISTERS, in the wgmma fragment layout: lane l of warp w
// holds rows r0 = 16w + l/4 and r1 = r0 + 8, and K positions q = l%4 and q + 4 of every k-step.  So each thread computes
// its own input features (enc_x entries q, q+4 mod 8 of both rows: ~10 accurate sinf per row; grid levels q, q+4, q+8, q+12
// of both rows) and a layer's accumulator fragment is the next layer's A operand without leaving the registers: the
// thread holds columns 8j + 2q, 8j + 2q + 1 of k-step j, so the packed weights take their K rows in that order
// (k_pack_tf32).  The bias + ReLU epilogues run on the fragments; the narrow outputs (deform 64->2, whose value IS
// `deform` and moves the canonical lookup; canonical 32->4 into the sigmoids) are fp32 dot products of the fragments,
// summed over the quad that shares the rows.  enc_x's A values are kept in shared memory (one column per thread) for the
// canonical net, whose K order [enc_x 42 | 0 x 6 | grid 32] starts with deform L0's.  Every row's arithmetic reads only
// that row, so a pixel's result does not depend on the other pixels of its tile or on the tile-to-CTA schedule.
// Budget: 112.5 KB of shared memory and <= 128 registers per thread, two CTAs (16 warps) per SM.
#include "common.cuh"
#include "launch.cuh"
#include "tc.cuh"
#include "torso_common.cuh"
#include "torso_kernel.cuh"

namespace gfpp {

using namespace torsoc;
using namespace tc;

namespace {

constexpr int TP = 128;    // pixels per tile
constexpr int NT = 256;
constexpr int NEX = 24;    // enc_x A values of a thread: 6 k-steps x 4

struct Smem {
    unsigned char w[TORSO_TF32_BYTES];   // tf32 hi / lo images of the wide layers (bulk copy; descriptors want 16-byte alignment)
    float ex[NEX][NT];                   // enc_x A values, one column per thread
    float wd2[2 * 64], wc2[4 * 32];
    float alpha[TP], col[3 * TP], dxy[2 * TP];
    int mask[TP];
    unsigned long long bar;
};

// freq_entry(x, 2, c) with the coordinate picked by a select: c depends on the lane here, and an indexed x would live in
// local memory.  Same operations, same value.
__device__ __forceinline__ float enc_x_entry(const float (&x)[2], int c) {
    const int d = c & 1;
    const float xd = d ? x[1] : x[0];
    if (c < 2) return xd;
    const int col = c / 2 - 1, f = col / 2;
    return sinf(__fadd_rn(scalbnf(xd, f), (float)(col % 2) * (3.141592653589793f / 2)));
}

// one k-step of A values -> tf32 hi / lo fragments
__device__ __forceinline__ void split_tf32(const float (&v)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        hi[e] = rna_tf32(v[e]);
        lo[e] = rna_tf32(v[e] - __uint_as_float(hi[e]));
    }
}

// ReLU(acc + bias) of an M = 64, N-wide accumulator fragment -> the next layer's A fragments (K order of k_pack_tf32)
template <int N>
__device__ __forceinline__ void relu_to_a(const float (&d)[N / 2], const float *__restrict__ bias, int q, uint32_t (&hi)[N / 8][4],
                                          uint32_t (&lo)[N / 8][4]) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
        const int c = 8 * j + 2 * q;
        const float b0 = bias ? __ldg(bias + c) : 0.f, b1 = bias ? __ldg(bias + c + 1) : 0.f;
        const float v[4] = {fmaxf(d[4 * j] + b0, 0.f), fmaxf(d[4 * j + 2] + b0, 0.f), fmaxf(d[4 * j + 1] + b1, 0.f),
                            fmaxf(d[4 * j + 3] + b1, 0.f)};
        split_tf32(v, hi[j], lo[j]);
    }
}

// O-wide fp32 output layer of ReLU(acc) (no bias): out[r][o] for the thread's rows r0 (r = 0) and r1 (r = 1); every lane of
// the quad ends with the same sums
template <int N, int O>
__device__ __forceinline__ void narrow_out(const float (&d)[N / 2], const float *__restrict__ w /*smem [O][N]*/, int q, float (&out)[2][O]) {
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int o = 0; o < O; ++o) out[r][o] = 0.f;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * q + e;
            const float h0 = fmaxf(d[4 * j + e], 0.f), h1 = fmaxf(d[4 * j + 2 + e], 0.f);
#pragma unroll
            for (int o = 0; o < O; ++o) {
                out[0][o] = fmaf(h0, w[o * N + c], out[0][o]);
                out[1][o] = fmaf(h1, w[o * N + c], out[1][o]);
            }
        }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int o = 0; o < O; ++o) {
            out[r][o] += __shfl_xor_sync(0xffffffffu, out[r][o], 1);
            out[r][o] += __shfl_xor_sync(0xffffffffu, out[r][o], 2);
        }
}

}  // namespace

// per-frame bias vectors: columns of the first deform / canonical layers that do not depend on the pixel
__global__ void k_torso_frame_bias(TorsoArgs a, const float *__restrict__ w_def0 /*[64,104]*/,
                                   const float *__restrict__ w_can0 /*[32,136]*/, const float *__restrict__ code,
                                   int code_dim, float *__restrict__ bias_def, float *__restrict__ bias_can) {
    const int f = blockIdx.x, j = threadIdx.x;
    __shared__ float h[64];
    const int n_pose = 6 + 6 * 2 * 4;  // 54
    if (j < n_pose) h[j] = freq_entry(a.pose6 + (size_t)f * 6, 6, j);
    else if (j < n_pose + code_dim) h[j] = code ? code[j - n_pose] : 0.f;
    __syncthreads();
    const int nh = n_pose + code_dim, din = 42 + nh;
    if (j < 64) {
        float s = 0.f;
        for (int k = 0; k < nh; ++k) s = fmaf(w_def0[j * din + 42 + k], h[k], s);
        bias_def[(size_t)f * 64 + j] = s;
    }
    if (j < 32) {
        float s = 0.f;
        for (int k = 0; k < nh; ++k) s = fmaf(w_can0[j * (32 + din) + 32 + 42 + k], h[k], s);
        bias_can[(size_t)f * 32 + j] = s;
    }
}

// MATTE: the composite tail also writes alpha_map / rgba_u8.  A compile-time switch, not a runtime branch: the kernel without it
// compiles to the same instructions as before the matte existed (a runtime branch reschedules the MMA section around it)
template <bool MATTE>
__device__ __forceinline__ void epilogue_body(const TorsoArgs &a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x;
    const int tiles_per_frame = (a.n_rays + TP - 1) / TP;
    const int n_tiles = a.n_frames * tiles_per_frame;
    if (a.has_torso) {
        if (tid == 0) {
            mbar_init(&s.bar, 1);
            mbar_fence_init();
            mbar_expect_tx(&s.bar, TORSO_TF32_BYTES);
            bulk_g2s(s.w, a.w_tf32, TORSO_TF32_BYTES, &s.bar);
        }
        for (int i = tid; i < 2 * 64; i += NT) s.wd2[i] = a.w_def2[i];
        for (int i = tid; i < 4 * 32; i += NT) s.wc2[i] = a.w_can2[i];
    }
    __syncthreads();
    bool w_ready = false;
    const int slot = tid & (TP - 1);
    // MMA-phase rows of this thread (tc.cuh: tf32 A fragment)
    const int r0 = 64 * (tid >> 7) + 16 * ((tid >> 5) & 3) + ((tid & 31) >> 2), r1 = r0 + 8;
    const uint32_t w_base = smem_u32(s.w);

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int f = tile / tiles_per_frame;
        const int n0 = (tile - f * tiles_per_frame) * TP;
        const int n = n0 + slot;
        const bool in_range = n < a.n_rays;
        int m = 0;
        if (a.has_torso && tid < TP && in_range) {
            const float occ = sample_density(a.density_grid_torso, a.grid_size, a.bg_coords[2 * n], a.bg_coords[2 * n + 1]);
            m = occ > a.density_thresh_torso ? 1 : 0;
        }
        if (tid < TP) s.mask[tid] = m;
        const int any = __syncthreads_or(m);
        if (any) {
            if (!w_ready) { mbar_wait(&s.bar, 0); w_ready = true; }
            // K position of the thread's A values, read here: hoisted out of the tile loop, the per-column constants derived
            // from it (frequency, phase, bias and weight offsets) would not fit the register budget beside the fragments
            int q;
            asm volatile("mov.u32 %0, %%laneid;" : "=r"(q));
            q &= 3;
            // x = shrink * bg_coord of rows r0, r1
            float x[2][2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int nr = n0 + (r ? r1 : r0);
                x[r][0] = x[r][1] = 0.f;
                if (nr < a.n_rays) { x[r][0] = __fmul_rn(a.bg_coords[2 * nr], a.torso_shrink); x[r][1] = __fmul_rn(a.bg_coords[2 * nr + 1], a.torso_shrink); }
            }
            // ---- deform net 104 -> 64 -> 64 -> 2 (radnerf_torso.py:60-76); L0's A = enc_x = freq10(x) [42 | 0 x 6] ----
            float dd[2][2];
            {
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    const int k0 = 8 * j + q, k1 = k0 + 4;
                    s.ex[4 * j][tid] = k0 < 42 ? enc_x_entry(x[0], k0) : 0.f;
                    s.ex[4 * j + 1][tid] = k0 < 42 ? enc_x_entry(x[1], k0) : 0.f;
                    s.ex[4 * j + 2][tid] = k1 < 42 ? enc_x_entry(x[0], k1) : 0.f;
                    s.ex[4 * j + 3][tid] = k1 < 42 ? enc_x_entry(x[1], k1) : 0.f;
                }
                // split after the sinf: the hi / lo fragments are not live across its slow path
                uint32_t ahi[6][4], alo[6][4];
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    const float ev[4] = {s.ex[4 * j][tid], s.ex[4 * j + 1][tid], s.ex[4 * j + 2][tid], s.ex[4 * j + 3][tid]};
                    split_tf32(ev, ahi[j], alo[j]);
                }
                float d[32];
                wgmma_tf32x3<64, 6>(d, ahi, alo, w_base + TORSO_TF32_D0.hi, w_base + TORSO_TF32_D0.hi + 64 * 48 * 4, 0u);
                wg_wait<0>();
                acc_fence(d);
                uint32_t hhi[8][4], hlo[8][4];
                relu_to_a<64>(d, a.bias_def + (size_t)f * 64, q, hhi, hlo);
                wgmma_tf32x3<64, 8>(d, hhi, hlo, w_base + TORSO_TF32_D1.hi, w_base + TORSO_TF32_D1.hi + 64 * 64 * 4, 0u);
                wg_wait<0>();
                acc_fence(d);
                narrow_out<64, 2>(d, s.wd2, q, dd);
            }
            // x = (x + dx).clamp(-1, 1)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                x[r][0] = fminf(fmaxf(x[r][0] + dd[r][0], -1.f), 1.f);
                x[r][1] = fminf(fmaxf(x[r][1] + dd[r][1], -1.f), 1.f);
            }
            if (q == 0) {
                s.dxy[r0] = dd[0][0]; s.dxy[TP + r0] = dd[0][1];
                s.dxy[r1] = dd[1][0]; s.dxy[TP + r1] = dd[1][1];
            }
            // ---- canonical net 136 -> 32 -> 32 -> 4, sigmoid (radnerf_torso.py:77-82); L0's A = [enc_x 42 | 0 x 6 | grid 32] ----
            {
                // K block [enc_x | 0 x 6] first: its MMAs run while the grid lookups below wait on memory
                float c[16];
                uint32_t ahi[6][4], alo[6][4];
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    const float ev[4] = {s.ex[4 * j][tid], s.ex[4 * j + 1][tid], s.ex[4 * j + 2][tid], s.ex[4 * j + 3][tid]};
                    split_tf32(ev, ahi[j], alo[j]);
                }
                wgmma_tf32x3<32, 6>(c, ahi, alo, w_base + TORSO_TF32_C0.hi, w_base + TORSO_TF32_C0.hi + 32 * 80 * 4, 0u);
                float u[2], v[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    u[r] = __fdiv_rn(__fadd_rn(x[r][0], 1.0f), 2.0f);
                    v[r] = __fdiv_rn(__fadd_rn(x[r][1], 1.0f), 2.0f);
                }
                uint32_t ghi[4][4], glo[4][4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {   // k-step 6 + j: level 4j + q, both features, of both rows
                    const float2 g0 = grid_lookup2(a.tor_gm, a.tor_tab, 4 * j + q, u[0], v[0]);
                    const float2 g1 = grid_lookup2(a.tor_gm, a.tor_tab, 4 * j + q, u[1], v[1]);
                    const float gv[4] = {g0.x, g1.x, g0.y, g1.y};
                    split_tf32(gv, ghi[j], glo[j]);
                }
                wgmma_tf32x3<32, 4>(c, ghi, glo, w_base + TORSO_TF32_C0.hi + 6 * 32 * 32, w_base + TORSO_TF32_C0.hi + 32 * 80 * 4 + 6 * 32 * 32, 1u);
                wg_wait<0>();
                acc_fence(c);
                uint32_t hhi[4][4], hlo[4][4];
                relu_to_a<32>(c, a.bias_can + (size_t)f * 32, q, hhi, hlo);
                wgmma_tf32x3<32, 4>(c, hhi, hlo, w_base + TORSO_TF32_C1.hi, w_base + TORSO_TF32_C1.hi + 32 * 32 * 4, 0u);
                wg_wait<0>();
                acc_fence(c);
                float o[2][4];
                narrow_out<32, 4>(c, s.wc2, q, o);
                if (q == 0) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int row = r ? r1 : r0;
                        s.alpha[row] = 1.0f / (1.0f + expf(-o[r][0]));
                        s.col[row] = 1.0f / (1.0f + expf(-o[r][1]));
                        s.col[TP + row] = 1.0f / (1.0f + expf(-o[r][2]));
                        s.col[2 * TP + row] = 1.0f / (1.0f + expf(-o[r][3]));
                    }
                }
            }
            __syncthreads();
        }
        // ---- composite (radnerf_torso.py:187-193 / renderer.py:386-392) ----
        if (tid < TP && in_range) {
            const size_t g = (size_t)f * a.n_rays + n;
            float ta = 0.f, tc[3] = {0.f, 0.f, 0.f}, dx = 0.f, dy = 0.f;
            if (any && s.mask[tid]) {
                ta = s.alpha[tid];
                tc[0] = s.col[tid]; tc[1] = s.col[TP + tid]; tc[2] = s.col[2 * TP + tid];
                dx = s.dxy[tid]; dy = s.dxy[TP + tid];
            }
            const float ws = a.wsum[g];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float bgc = a.bg_color ? a.bg_color[3 * (size_t)n + c] : 1.0f;
                // bg = torso_color * alpha + bg * (1 - alpha); image = image + (1 - ws) * bg; clamp(0, 1)
                const float bg = a.has_torso ? __fadd_rn(__fmul_rn(tc[c], ta), __fmul_rn(bgc, __fsub_rn(1.0f, ta))) : bgc;
                const float v = __fadd_rn(a.image[3 * g + c], __fmul_rn(__fsub_rn(1.0f, ws), bg));
                const float vc = fminf(fmaxf(v, 0.f), 1.f);
                if (a.rgb_map) a.rgb_map[3 * g + c] = vc;
                // (rgb * 255).int() -> uint8: what the driver hands the video writer (genefacepp_infer.py:469, 505)
                if (a.rgb_u8) a.rgb_u8[3 * g + c] = (unsigned char)(int)__fmul_rn(vc, 255.0f);
                if (a.torso_rgb) a.torso_rgb[3 * g + c] = bg;
            }
            // the matte: premultiplied P = clamp(image + (1 - ws) * (torso_color * alpha)) and coverage A = ws + (1 - ws) * alpha,
            // without the background, so that P + (1 - A) * B is the frame over any B (bg = 0 above gives the same P bits)
            if constexpr (MATTE) {
                const float A = __fadd_rn(ws, __fmul_rn(__fsub_rn(1.0f, ws), ta));
                if (a.alpha_map) a.alpha_map[g] = A;
                if (a.rgba_u8) {
                    uint32_t px = (uint32_t)(unsigned char)(int)__fmul_rn(A, 255.0f) << 24;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float p = __fadd_rn(a.image[3 * g + c], __fmul_rn(__fsub_rn(1.0f, ws), __fmul_rn(tc[c], ta)));
                        px |= (uint32_t)(unsigned char)(int)__fmul_rn(fminf(fmaxf(p, 0.f), 1.f), 255.0f) << (8 * c);
                    }
                    reinterpret_cast<uint32_t *>(a.rgba_u8)[g] = px;   // one 32-bit store per pixel: the warp's stores coalesce
                }
            }
            if (a.torso_alpha) a.torso_alpha[g] = ta;
            if (a.deform) { a.deform[2 * g] = dx; a.deform[2 * g + 1] = dy; }
            if (a.P_count && any && s.mask[tid]) atomicAdd(a.P_count + f, 1);
        }
        __syncthreads();
    }
    // the weight copy must land before the CTA exits, also when none of its tiles had a torso pixel: its shared memory is
    // released at exit and may already belong to the next CTA on this SM
    if (a.has_torso && !w_ready) mbar_wait(&s.bar, 0);
}

__global__ void __launch_bounds__(256, 2) k_epilogue(const __grid_constant__ TorsoArgs a) { epilogue_body<false>(a); }
__global__ void __launch_bounds__(256, 2) k_epilogue_matte(const __grid_constant__ TorsoArgs a) { epilogue_body<true>(a); }

// dst[k][n] = src[(row0 + n) * ld + col0 + k] for k < K, zero for K <= k < Kpad   (k-major repack of nn.Linear weights)
__global__ void k_pack_kmajor(const float *__restrict__ src, int ld, int row0, int col0, int N, int K, int Kpad,
                              float *__restrict__ dst) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Kpad * N; i += gridDim.x * blockDim.x) {
        const int k = i / N, n = i - k * N;
        dst[i] = k < K ? src[(size_t)(row0 + n) * ld + col0 + k] : 0.f;
    }
}

// source column of K position k of tf32 torso layer `layer` (0 deform L0, 1 deform L1, 2 canonical L0, 3 canonical L1), -1 for
// a zero row.  Accumulator-fragment order inside every 8 (the grid block and the hidden layers): position p < 4 takes column
// 2p, position p >= 4 takes column 2(p - 4) + 1.
__device__ __forceinline__ int tf32_src_col(int layer, int k) {
    const int p = k & 7, perm = (k & ~7) + (p < 4 ? 2 * p : 2 * p - 7);
    if (layer == 0) return k < 42 ? k : -1;
    if (layer == 2) return k < 42 ? 32 + k : k < 48 ? -1 : perm - 48;   // [enc_x = source columns 32..73 | 0 x 6 | grid 0..31]
    return perm;
}

// tf32 hi / lo images of the four wide torso layers (torso_kernel.cuh layout) from the nn.Linear weights [out, in]
__global__ void k_pack_tf32(const float *__restrict__ w_def0, int ld_def0, const float *__restrict__ w_def1,
                            const float *__restrict__ w_can0, int ld_can0, const float *__restrict__ w_can1, unsigned char *__restrict__ dst) {
    constexpr int n_el = 64 * 48 + 64 * 64 + 32 * 80 + 32 * 32;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_el; i += gridDim.x * blockDim.x) {
        int layer = 0, r = i, N = 64, K = 48, hi = TORSO_TF32_D0.hi, ld = ld_def0;
        const float *src = w_def0;
        if (r >= 64 * 48) { r -= 64 * 48; layer = 1; K = 64; hi = TORSO_TF32_D1.hi; ld = 64; src = w_def1;
            if (r >= 64 * 64) { r -= 64 * 64; layer = 2; N = 32; K = 80; hi = TORSO_TF32_C0.hi; ld = ld_can0; src = w_can0;
                if (r >= 32 * 80) { r -= 32 * 80; layer = 3; K = 32; hi = TORSO_TF32_C1.hi; ld = 32; src = w_can1; } } }
        const int n = r / K, k = r - n * K;
        const int c = tf32_src_col(layer, k);
        const float w = c >= 0 ? src[(size_t)n * ld + c] : 0.f;
        const uint32_t h = rna_tf32(w), l = rna_tf32(w - __uint_as_float(h));
        const uint32_t off = (uint32_t)((k >> 3) * N * 32) + k16_off(n, (k & 7) >> 2) + 4u * (uint32_t)(k & 3);
        *reinterpret_cast<uint32_t *>(dst + hi + off) = h;
        *reinterpret_cast<uint32_t *>(dst + hi + N * K * 4 + off) = l;
    }
}

// dst[o][k] = src[(row0 + o) * ld + k]   (plain row copy for the narrow output layers)
__global__ void k_pack_rows(const float *__restrict__ src, int ld, int row0, int n_rows, int K, int dst_ld,
                            float *__restrict__ dst) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rows * K; i += gridDim.x * blockDim.x) {
        const int o = i / K, k = i - o * K;
        dst[o * dst_ld + k] = src[(size_t)(row0 + o) * ld + k];
    }
}

// bias[n] = sum_k W[n][col0 + k] * v[k]   (folds a per-model constant input block into a bias)
__global__ void k_fold_bias(const float *__restrict__ W, int ld, int col0, int nk, const float *__restrict__ v, int N,
                            float *__restrict__ bias) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float s = 0.f;
    for (int k = 0; k < nk; ++k) s = fmaf(W[(size_t)n * ld + col0 + k], v ? v[k] : 0.f, s);
    bias[n] = s;
}

size_t epilogue_smem_bytes() { return sizeof(Smem); }

cudaError_t launch_torso_frame_bias(const TorsoArgs &a, const float *w_def0, const float *w_can0, const float *code,
                                    int code_dim, float *bias_def, float *bias_can, cudaStream_t st) {
    k_torso_frame_bias<<<a.n_frames, 64, 0, st>>>(a, w_def0, w_can0, code, code_dim, bias_def, bias_can);
    return cudaGetLastError();
}

cudaError_t launch_epilogue(const TorsoArgs &a, cudaStream_t st) {
    // function attributes are per device: set on every launch (a few microseconds), never cached process-wide
    const auto kernel = a.alpha_map || a.rgba_u8 ? k_epilogue_matte : k_epilogue;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    const int tiles = a.n_frames * ((a.n_rays + TP - 1) / TP);
    int blocks = 2 * sm_count();
    if (tiles < blocks) blocks = tiles > 0 ? tiles : 1;
    kernel<<<blocks, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_pack_kmajor(const float *src, int ld, int row0, int col0, int N, int K, int Kpad, float *dst, cudaStream_t st) {
    k_pack_kmajor<<<grid_for((uint64_t)Kpad * N, 256), 256, 0, st>>>(src, ld, row0, col0, N, K, Kpad, dst);
    return cudaGetLastError();
}
cudaError_t launch_pack_tf32(const float *w_def0, int ld_def0, const float *w_def1, const float *w_can0, int ld_can0,
                             const float *w_can1, unsigned char *dst, cudaStream_t st) {
    k_pack_tf32<<<grid_for(64 * 48 + 64 * 64 + 32 * 80 + 32 * 32, 256), 256, 0, st>>>(w_def0, ld_def0, w_def1, w_can0, ld_can0, w_can1, dst);
    return cudaGetLastError();
}
cudaError_t launch_pack_rows(const float *src, int ld, int row0, int n_rows, int K, int dst_ld, float *dst, cudaStream_t st) {
    k_pack_rows<<<grid_for((uint64_t)n_rows * K, 256), 256, 0, st>>>(src, ld, row0, n_rows, K, dst_ld, dst);
    return cudaGetLastError();
}
cudaError_t launch_fold_bias(const float *W, int ld, int col0, int nk, const float *v, int N, float *bias, cudaStream_t st) {
    k_fold_bias<<<(N + 127) / 128, 128, 0, st>>>(W, ld, col0, nk, v, N, bias);
    return cudaGetLastError();
}

}  // namespace gfpp
