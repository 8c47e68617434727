// torso_sr_train_kernel.cu -- RADNeRFTorsowithSR.forward_torso (modules/radnerfs/radnerf_torso_sr.py:75-114) with its gradient, fp32 FFMA.
//
//   h = [freq10(shrink * x) 42 | code | freq4(jaw lm68) 126 | head-aware 16] -> deform net (din -> 64 -> 64 -> 2) -> dx
//   x2 = clamp(shrink * x + dx, -1, 1);  [tiled 2-D grid at (x2 + 1) / 2 | h] -> canonical net (32 + din -> 32 -> 32 -> 4) -> sigmoid
//   head-aware = head_color_weights_encoder(cat[image, weights_sum]): 4 -> 16 -> 32 -> 16 with biases, LeakyReLU(0.02)
//
// Shape of the computation
//   * the constant columns of both first layers ([code | freq4(jaw)]) are folded into bias vectors and the weights are laid out
//     k-major by k_torso_sr_field_relayout, into the caller's workspace, exactly as gfpp_torso_sr_pack + k_torso_sr_frame_bias lay
//     them out for the render epilogue: the forward IS k_torso_sr's field (its point mode, torso_sr_kernel.cu) on that workspace, so
//     it is bit-identical to the composite's torso_alpha_map and torso_deform at the same parameters and inputs;
//   * k_torso_sr_field_bwd recomputes the forward of its 128-point tile with the same tile GEMMs (small_gemm / store_relu) and the same
//     head-aware encoder arithmetic in the same operation order -- its ReLU, LeakyReLU and clamp decisions are those of the forward --
//     keeps every activation in shared memory, and then runs the whole backward; no per-point state is saved between the calls;
//   * the head-aware encoding enters both first layers: its gradient is the sum of their 16 encoding columns' input gradients, which
//     then goes back through the encoder (LeakyReLU' from the recomputed activations) to its three weights and biases;
//   * the constant columns' weight gradients and the code's gradient follow from the column sums of the two first layers' output
//     gradients (k_torso_sr_field_reduce); the landmarks get no gradient;
//   * weight gradients: each persistent CTA owns a contiguous range of tiles and a block of partial sums in the workspace that its
//     threads update with plain read-modify-writes (each element has one owner thread); k_torso_sr_field_reduce sums the blocks in
//     CTA order.  Only the table gradient depends on scheduling: it is scattered with float2 vector reductions (grid_train.cuh).
#include "grid_train.cuh"
#include "launch.cuh"
#include "torso_common.cuh"
#include "torso_sr_train_kernel.cuh"

namespace gfpp {

using namespace torsoc;

namespace {

constexpr int TP = TORSO_SR_TRAIN_TP;
constexpr int NT = 256;
constexpr int KD0 = TORSO_SR_KD0, KC0 = TORSO_SR_KC0;   // 60, 92
constexpr int LDC = 100;   // CI row stride: canonical input [grid 32 | enc_x 42 | head-aware 16 | 0 0]; CI + 32 is the deform input
constexpr int LDH = 68;    // deform hidden rows
constexpr int LDS = 36;    // canonical hidden rows
constexpr int LDG = 16;    // gradient of the head-aware encoding
constexpr int NJAW = 14, NLM = NJAW + NJAW * 2 * 4;   // 126

struct Smem {
    float CI[TP * LDC];
    float H1[TP * LDH];
    float H2[TP * LDH];
    float C1[TP * LDS];
    float C2[TP * LDS];
    float GHA[TP * LDG];
    float wd0[KD0 * 64], wd1[64 * 64], wc0[KC0 * 32], wc1[32 * 32];
    float wd2[2 * 64], wc2[4 * 32];
    float ha[TORSO_SR_HA_FLOATS];
    float xs[2 * TP];        // shrink * x
    float v[2 * TP];         // shrink * x + dx, before the clamp
    float g4[TP * 4];        // gradient of the canonical logits
    float gx[TP * 2];        // gradient of dx
    float gin[2 * TP * 2];   // grid input gradient, one partial per level group
};

__device__ __forceinline__ float leaky002(float x) { return x > 0.f ? x : 0.02f * x; }

// head_color_weights_encoder of one point in k_torso_sr's operation order: h1 = LeakyReLU(L0), h2 = L1 (before its LeakyReLU), o = L2
__device__ __forceinline__ void ha_encode(const float *ha, const float (&in4)[4], float (&h1)[16], float (&h2)[32]) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        float t = ha[TORSO_SR_HA_B0 + j];
#pragma unroll
        for (int k = 0; k < 4; ++k) t = fmaf(in4[k], ha[TORSO_SR_HA_W0 + k * 16 + j], t);
        h1[j] = leaky002(t);
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) h2[j] = ha[TORSO_SR_HA_B1 + j];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
#pragma unroll
        for (int j = 0; j < 32; ++j) h2[j] = fmaf(h1[k], ha[TORSO_SR_HA_W1 + k * 32 + j], h2[j]);
    }
}

__device__ __forceinline__ void ha_input(const TorsoSrTrainArgs &a, uint32_t p, bool in_range, float (&in4)[4]) {
    in4[0] = in4[1] = in4[2] = in4[3] = 0.f;
    if (in_range && a.image) {
        in4[0] = a.image[3 * (size_t)p]; in4[1] = a.image[3 * (size_t)p + 1]; in4[2] = a.image[3 * (size_t)p + 2]; in4[3] = a.wsum[p];
    }
}

// part[n][c] += sum_p Y[p][n] * X[p][c] for n < N, c < C (multiples of 4), p over the tile in order; one thread per 4x4 block,
// so every element has one owner thread and the read-modify-write needs no atomics.
template <int N, int C>
__device__ __forceinline__ void wgrad(const float *Y, int ldy, const float *X, int ldx, float *__restrict__ part, int ldp, int tid) {
    constexpr int CB = C / 4, NBLK = (N / 4) * CB;
    for (int b = tid; b < NBLK; b += NT) {
        const int n0 = (b / CB) * 4, c0 = (b % CB) * 4;
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
        for (int p = 0; p < TP; ++p) {
            const float4 y = *reinterpret_cast<const float4 *>(Y + p * ldy + n0);
            const float4 x = *reinterpret_cast<const float4 *>(X + p * ldx + c0);
            const float yv[4] = {y.x, y.y, y.z, y.w}, xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(yv[i], xv[j], acc[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) part[(size_t)(n0 + i) * ldp + c0 + j] += acc[i][j];
    }
}

// Input gradient of a layer: out[p][k] = sum_o G[p][o] * WT[k][o] for k < K, WT the k-major weights ([in][out] = W^T).  With MASK
// it goes through the ReLU whose output `out` holds: zero where out[p][k] <= 0 (in place; each element has one owner thread).
template <int NO, int K, bool MASK>
__device__ __forceinline__ void dgrad(const float *G, int ldg, const float *WT, float *out, int ldo, int tid) {
    const int p = tid & (TP - 1), kh = tid >> 7;
    float g[NO];
#pragma unroll
    for (int o = 0; o < NO; o += 4) {
        const float4 t = *reinterpret_cast<const float4 *>(G + p * ldg + o);
        g[o] = t.x; g[o + 1] = t.y; g[o + 2] = t.z; g[o + 3] = t.w;
    }
    for (int k = kh; k < K; k += NT / TP) {
        float v = 0.f;
#pragma unroll
        for (int o = 0; o < NO; ++o) v = fmaf(g[o], WT[k * NO + o], v);
        if (MASK && !(out[p * ldo + k] > 0.f)) v = 0.f;
        out[p * ldo + k] = v;
    }
}

// Input gradient of a head-aware layer through the LeakyReLU whose output act[p][k] holds (PyTorch's rule: slope 1 where the
// output is > 0, else 0.02): out[p][k] = sum_o G[p][o] * WT[k][o] (* 0.02), k < K.
template <int NO, int K>
__device__ __forceinline__ void dgrad_leaky(const float *G, int ldg, const float *WT, const float *act, int lda, float *out, int ldo, int tid) {
    for (int e = tid; e < TP * K; e += NT) {
        const int q = e / K, k = e % K;
        float v = 0.f;
#pragma unroll
        for (int o = 0; o < NO; ++o) v = fmaf(G[q * ldg + o], WT[k * NO + o], v);
        out[q * ldo + k] = act[q * lda + k] > 0.f ? v : v * 0.02f;
    }
}

// column sums over the tile: part[n] += sum_p Y[p][n], n < N
template <int N>
__device__ __forceinline__ void colsum(const float *Y, int ldy, float *__restrict__ part, int tid) {
    if (tid < N) {
        float v = 0.f;
        for (int p = 0; p < TP; ++p) v += Y[p * ldy + tid];
        part[tid] += v;
    }
}

// entry j of the constant block [code | freq4(jaw)] of both first layers, as k_torso_sr_frame_bias forms it
__device__ __forceinline__ float const_col(const TorsoSrTrainArgs &a, int j) {
    return j < a.code_dim ? (a.code ? a.code[j] : 0.f) : freq_entry(a.lm68 + 10, NJAW, j - a.code_dim);   // points 5..11 of [68,2]
}

}  // namespace

// The forward's workspace (TorsoSrWt), one thread per output float: the k-major copies gfpp_torso_sr_pack makes of the weights and
// the head-aware encoder, and the biases k_torso_sr_frame_bias folds for one frame, in their operation order.
__global__ void k_torso_sr_field_relayout(const __grid_constant__ TorsoSrTrainArgs a) {
    const int nh = a.code_dim + NLM, din = 42 + nh + (a.head_aware ? 16 : 0), ldc = 32 + din;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < (uint32_t)TorsoSrWt::total; i += gridDim.x * blockDim.x) {
        float v = 0.f;
        if (i >= TorsoSrWt::bias_can) {
            const uint32_t j = i - (uint32_t)TorsoSrWt::bias_can;
            for (int k = 0; k < nh; ++k) v = fmaf(a.w_can[0][j * ldc + 32 + 42 + k], const_col(a, k), v);
        } else if (i >= TorsoSrWt::bias_def) {
            const uint32_t j = i - (uint32_t)TorsoSrWt::bias_def;
            for (int k = 0; k < nh; ++k) v = fmaf(a.w_def[0][j * din + 42 + k], const_col(a, k), v);
        } else if (i >= TorsoSrWt::ha) {
            const uint32_t r = i - (uint32_t)TorsoSrWt::ha;
            if (a.head_aware) {
                if (r >= TORSO_SR_HA_B2) v = a.ha_b[2][r - TORSO_SR_HA_B2];
                else if (r >= TORSO_SR_HA_W2) { const uint32_t q = r - TORSO_SR_HA_W2; v = a.ha_w[2][(q % 16) * 32 + q / 16]; }
                else if (r >= TORSO_SR_HA_B1) v = a.ha_b[1][r - TORSO_SR_HA_B1];
                else if (r >= TORSO_SR_HA_W1) { const uint32_t q = r - TORSO_SR_HA_W1; v = a.ha_w[1][(q % 32) * 16 + q / 32]; }
                else if (r >= TORSO_SR_HA_B0) v = a.ha_b[0][r - TORSO_SR_HA_B0];
                else v = a.ha_w[0][(r % 16) * 4 + r / 16];
            }
        } else if (i >= TorsoSrWt::wc2) {
            v = a.w_can[2][i - TorsoSrWt::wc2];
        } else if (i >= TorsoSrWt::wc1) {
            const uint32_t r = i - (uint32_t)TorsoSrWt::wc1, k = r / 32, n = r % 32;
            v = a.w_can[1][n * 32 + k];
        } else if (i >= TorsoSrWt::wc0) {
            const uint32_t r = i - (uint32_t)TorsoSrWt::wc0, k = r / 32, n = r % 32;
            if (k < 74) v = a.w_can[0][n * ldc + k];
            else if (k < 90 && a.head_aware) v = a.w_can[0][n * ldc + 74 + nh + (k - 74)];
        } else if (i >= TorsoSrWt::wd2) {
            v = a.w_def[2][i - TorsoSrWt::wd2];
        } else if (i >= TorsoSrWt::wd1) {
            const uint32_t r = i - (uint32_t)TorsoSrWt::wd1, k = r / 64, n = r % 64;
            v = a.w_def[1][n * 64 + k];
        } else {
            const uint32_t k = i / 64, n = i % 64;
            if (k < 42) v = a.w_def[0][n * din + k];
            else if (k < 58 && a.head_aware) v = a.w_def[0][n * din + 42 + nh + (k - 42)];
        }
        a.wt[i] = v;
    }
}

// Per tile: the forward in k_torso_sr's operation order, then
//   1 sigmoid' -> g4;  2 dW can2, g_c2 in place (C2);  3 dW can1, g_c1 in place (C1);  4 dW can0, column sums, g_grid -> C2,
//     g_ha (canonical columns) -> GHA;  5 grid: table scatter, input gradient through dy_dx, (x+1)/2, clamp mask, + g_deform -> gx;
//   6 dW def2, g_h2 in place (H2);  7 dW def1, g_h1 in place (H1);  8 dW def0, column sums, GHA += g_ha (deform columns);
//   9 head-aware encoder: recomputed activations -> H2, dW/db L2, g -> C1, dW/db L1, g -> C2, dW/db L0
__global__ void __launch_bounds__(NT, 1) k_torso_sr_field_bwd(const __grid_constant__ TorsoSrTrainArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x;
    const bool ha_on = a.head_aware != 0;
    float *part = a.part + (size_t)blockIdx.x * TorsoSrPart::total;
    for (size_t i = tid; i < TorsoSrPart::total; i += NT) part[i] = 0.f;
    for (int i = tid; i < KD0 * 64; i += NT) s.wd0[i] = a.wt[TorsoSrWt::wd0 + i];
    for (int i = tid; i < 64 * 64; i += NT) s.wd1[i] = a.wt[TorsoSrWt::wd1 + i];
    for (int i = tid; i < KC0 * 32; i += NT) s.wc0[i] = a.wt[TorsoSrWt::wc0 + i];
    for (int i = tid; i < 32 * 32; i += NT) s.wc1[i] = a.wt[TorsoSrWt::wc1 + i];
    for (int i = tid; i < 2 * 64; i += NT) s.wd2[i] = a.wt[TorsoSrWt::wd2 + i];
    for (int i = tid; i < 4 * 32; i += NT) s.wc2[i] = a.wt[TorsoSrWt::wc2 + i];
    for (int i = tid; i < TORSO_SR_HA_FLOATS; i += NT) s.ha[i] = a.wt[TorsoSrWt::ha + i];
    __syncthreads();
    const int ty = tid >> 4, tx = tid & 15;
    const int slot = tid & (TP - 1), lg = tid >> 7;
    const uint32_t n_tiles = (a.M + TP - 1) / TP;
    const uint32_t t0 = (uint32_t)((uint64_t)n_tiles * blockIdx.x / gridDim.x), t1 = (uint32_t)((uint64_t)n_tiles * (blockIdx.x + 1) / gridDim.x);
    for (uint32_t tile = t0; tile < t1; ++tile) {
        const uint32_t p = tile * TP + slot;
        const bool in_range = p < a.M;
        // ---- forward: [enc_x | head-aware encoding | 0 0] -> CI[:, 32:92] ----
        {
            float x[2] = {0.f, 0.f};
            if (in_range) { x[0] = __fmul_rn(a.xy[2 * (size_t)p], a.shrink); x[1] = __fmul_rn(a.xy[2 * (size_t)p + 1], a.shrink); }
            for (int c = lg * 30; c < lg * 30 + 30; ++c) {
                if (c >= 42 && c < 58) continue;
                s.CI[slot * LDC + 32 + c] = c < 42 ? freq_entry(x, 2, c) : 0.f;
            }
            if (lg == 0) {
                s.xs[slot] = x[0]; s.xs[TP + slot] = x[1];
                float o[16];
                if (ha_on) {
                    float in4[4], h1[16], h2[32];
                    ha_input(a, p, in_range, in4);
                    ha_encode(s.ha, in4, h1, h2);
#pragma unroll
                    for (int j = 0; j < 16; ++j) o[j] = s.ha[TORSO_SR_HA_B2 + j];
#pragma unroll
                    for (int k = 0; k < 32; ++k) {
                        const float hk = leaky002(h2[k]);
#pragma unroll
                        for (int j = 0; j < 16; ++j) o[j] = fmaf(hk, s.ha[TORSO_SR_HA_W2 + k * 16 + j], o[j]);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j) o[j] = 0.f;
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) s.CI[slot * LDC + 74 + j] = o[j];
            }
        }
        __syncthreads();
        {
            float acc[8][4] = {};
            small_gemm<4, KD0, LDC>(acc, s.CI + 32, s.wd0, ty, tx);
            store_relu<4, LDH>(acc, s.H1, a.wt + TorsoSrWt::bias_def, ty, tx);
        }
        __syncthreads();
        {
            float acc[8][4] = {};
            small_gemm<4, 64, LDH>(acc, s.H1, s.wd1, ty, tx);
            store_relu<4, LDH>(acc, s.H2, nullptr, ty, tx);
        }
        __syncthreads();
        {
            const int row = tid >> 1, half = tid & 1;
            float v0 = 0.f, v1 = 0.f;
            for (int k = half * 32; k < half * 32 + 32; ++k) {
                const float xk = s.H2[row * LDH + k];
                v0 = fmaf(xk, s.wd2[k], v0);
                v1 = fmaf(xk, s.wd2[64 + k], v1);
            }
            v0 += __shfl_xor_sync(0xffffffffu, v0, 1);
            v1 += __shfl_xor_sync(0xffffffffu, v1, 1);
            if (half == 0) { s.v[row] = s.xs[row] + v0; s.v[TP + row] = s.xs[TP + row] + v1; }
        }
        __syncthreads();
        float u[2];
        u[0] = __fdiv_rn(__fadd_rn(fminf(fmaxf(s.v[slot], -1.f), 1.f), 1.0f), 2.0f);
        u[1] = __fdiv_rn(__fadd_rn(fminf(fmaxf(s.v[TP + slot], -1.f), 1.f), 1.0f), 2.0f);
#pragma unroll 2
        for (int l = lg * 8; l < lg * 8 + 8; ++l)
            *reinterpret_cast<float2 *>(s.CI + slot * LDC + 2 * l) = grid_lookup2(a.gm, a.tab, l, u[0], u[1]);
        __syncthreads();
        {
            float acc[8][2] = {};
            small_gemm<2, KC0, LDC>(acc, s.CI, s.wc0, ty, tx);
            store_relu<2, LDS>(acc, s.C1, a.wt + TorsoSrWt::bias_can, ty, tx);
        }
        __syncthreads();
        {
            float acc[8][2] = {};
            small_gemm<2, 32, LDS>(acc, s.C1, s.wc1, ty, tx);
            store_relu<2, LDS>(acc, s.C2, nullptr, ty, tx);
        }
        __syncthreads();
        // ---- 1: canonical logits, sigmoid' ----
        {
            const int row = tid >> 1, half = tid & 1;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            for (int k = half * 16; k < half * 16 + 16; ++k) {
                const float xk = s.C2[row * LDS + k];
#pragma unroll
                for (int o = 0; o < 4; ++o) v[o] = fmaf(xk, s.wc2[o * 32 + k], v[o]);
            }
#pragma unroll
            for (int o = 0; o < 4; ++o) v[o] += __shfl_xor_sync(0xffffffffu, v[o], 1);
            const uint32_t pr = tile * TP + row;
            if (half == 0) {
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    const float y = 1.0f / (1.0f + expf(-v[o]));
                    const float g = pr < a.M ? (o == 0 ? a.g_alpha[pr] : a.g_color[3 * (size_t)pr + o - 1]) : 0.f;
                    s.g4[row * 4 + o] = g * (1.0f - y) * y;
                }
            }
        }
        __syncthreads();
        // ---- 2 ----
        if (tid < 128) {
            const int o = tid >> 5, k = tid & 31;
            float v = 0.f;
            for (int q = 0; q < TP; ++q) v = fmaf(s.g4[q * 4 + o], s.C2[q * LDS + k], v);
            part[TorsoSrPart::c2 + tid] += v;
        }
        __syncthreads();
        for (int e = tid; e < TP * 32; e += NT) {
            const int q = e >> 5, k = e & 31;
            float v = 0.f;
#pragma unroll
            for (int o = 0; o < 4; ++o) v = fmaf(s.g4[q * 4 + o], s.wc2[o * 32 + k], v);
            s.C2[q * LDS + k] = s.C2[q * LDS + k] > 0.f ? v : 0.f;
        }
        __syncthreads();
        // ---- 3 ----
        wgrad<32, 32>(s.C2, LDS, s.C1, LDS, part + TorsoSrPart::c1, 32, tid);
        __syncthreads();
        dgrad<32, 32, true>(s.C2, LDS, s.wc1, s.C1, LDS, tid);
        __syncthreads();
        // ---- 4 ----
        wgrad<32, KC0>(s.C1, LDS, s.CI, LDC, part + TorsoSrPart::c0, KC0, tid);
        if (tid >= 224) colsum<32>(s.C1, LDS, part + TorsoSrPart::csc, tid - 224);
        dgrad<32, 32, false>(s.C1, LDS, s.wc0, s.C2, LDS, tid);
        if (ha_on) dgrad<32, 16, false>(s.C1, LDS, s.wc0 + 74 * 32, s.GHA, LDG, tid);
        __syncthreads();
        // ---- 5: grid -- table gradient, input gradient through dy_dx and the (x+1)/2 map, clamp, + g_deform ----
        {
            float gin[3] = {0.f, 0.f, 0.f};
            if (in_range) {
                for (int l = lg * 8; l < lg * 8 + 8; ++l) {
                    const float2 g = *reinterpret_cast<const float2 *>(s.C2 + slot * LDS + 2 * l);
                    grid_scatter<2>(a.gm, l, u, g, a.g_tab);
                    grid_input_grad<2>(a.gm, a.tab, l, u, g, gin);
                }
            }
            s.gin[(lg * TP + slot) * 2] = gin[0];
            s.gin[(lg * TP + slot) * 2 + 1] = gin[1];
        }
        __syncthreads();
        if (tid < TP) {
#pragma unroll
            for (int d = 0; d < 2; ++d) {
                float g = 0.f;
                if (in_range) {
                    // levels 0..7 then 8..15, then the 1/2 of (x + 1) / 2; clamp(-1, 1) passes the gradient on [-1, 1] inclusive
                    const float vd = s.v[d * TP + tid];
                    const float gl = (s.gin[tid * 2 + d] + s.gin[(TP + tid) * 2 + d]) / 2.0f;
                    g = (vd >= -1.f && vd <= 1.f ? gl : 0.f) + a.g_deform[2 * (size_t)p + d];
                }
                s.gx[tid * 2 + d] = g;
            }
        }
        __syncthreads();
        // ---- 6 ----
        if (tid < 128) {
            const int o = tid >> 6, k = tid & 63;
            float v = 0.f;
            for (int q = 0; q < TP; ++q) v = fmaf(s.gx[q * 2 + o], s.H2[q * LDH + k], v);
            part[TorsoSrPart::d2 + tid] += v;
        }
        __syncthreads();
        for (int e = tid; e < TP * 64; e += NT) {
            const int q = e >> 6, k = e & 63;
            const float v = fmaf(s.gx[q * 2 + 1], s.wd2[64 + k], s.gx[q * 2] * s.wd2[k]);
            s.H2[q * LDH + k] = s.H2[q * LDH + k] > 0.f ? v : 0.f;
        }
        __syncthreads();
        // ---- 7 ----
        wgrad<64, 64>(s.H2, LDH, s.H1, LDH, part + TorsoSrPart::d1, 64, tid);
        __syncthreads();
        dgrad<64, 64, true>(s.H2, LDH, s.wd1, s.H1, LDH, tid);
        __syncthreads();
        // ---- 8 ----
        wgrad<64, KD0>(s.H1, LDH, s.CI + 32, LDC, part + TorsoSrPart::d0, KD0, tid);
        if (tid >= 192) colsum<64>(s.H1, LDH, part + TorsoSrPart::csd, tid - 192);
        if (ha_on) {
            for (int e = tid; e < TP * 16; e += NT) {
                const int q = e >> 4, j = e & 15;
                float v = s.GHA[q * LDG + j];
                for (int n = 0; n < 64; ++n) v = fmaf(s.H1[q * LDH + n], s.wd0[(42 + j) * 64 + n], v);
                s.GHA[q * LDG + j] = v;
            }
        }
        __syncthreads();
        // ---- 9: head-aware encoder ----
        if (ha_on) {
            if (tid < TP) {
                float in4[4], h1[16], h2[32];
                ha_input(a, p, in_range, in4);
                ha_encode(s.ha, in4, h1, h2);
#pragma unroll
                for (int j = 0; j < 16; ++j) s.H2[tid * LDH + j] = h1[j];
#pragma unroll
                for (int j = 0; j < 32; ++j) s.H2[tid * LDH + 16 + j] = leaky002(h2[j]);
#pragma unroll
                for (int j = 0; j < 4; ++j) s.H2[tid * LDH + 48 + j] = in4[j];
            }
            __syncthreads();
            wgrad<16, 32>(s.GHA, LDG, s.H2 + 16, LDH, part + TorsoSrPart::hw2, 32, tid);
            if (tid >= 224) colsum<16>(s.GHA, LDG, part + TorsoSrPart::hb2, tid - 224);
            dgrad_leaky<16, 32>(s.GHA, LDG, s.ha + TORSO_SR_HA_W2, s.H2 + 16, LDH, s.C1, LDS, tid);
            __syncthreads();
            wgrad<32, 16>(s.C1, LDS, s.H2, LDH, part + TorsoSrPart::hw1, 16, tid);
            if (tid >= 224) colsum<32>(s.C1, LDS, part + TorsoSrPart::hb1, tid - 224);
            dgrad_leaky<32, 16>(s.C1, LDS, s.ha + TORSO_SR_HA_W1, s.H2, LDH, s.C2, LDS, tid);
            __syncthreads();
            wgrad<16, 4>(s.C2, LDS, s.H2 + 48, LDH, part + TorsoSrPart::hw0, 4, tid);
            if (tid >= 224) colsum<16>(s.C2, LDS, part + TorsoSrPart::hb0, tid - 224);
            __syncthreads();
        }
    }
}

// Sums the per-CTA partials in CTA order into the caller's gradient buffers; the constant columns of both first layers and the
// code's gradient follow from the column sums.  blockIdx.y selects the output.
__global__ void k_torso_sr_field_reduce(const __grid_constant__ TorsoSrTrainArgs a) {
    const int seg = blockIdx.y;
    const uint32_t G = a.n_cta;
    const size_t P = TorsoSrPart::total;
    auto sum = [&](size_t off) {
        float v = 0.f;
        for (uint32_t c = 0; c < G; ++c) v += a.part[c * P + off];
        return v;
    };
    const int nh = a.code_dim + NLM, din = 42 + nh + (a.head_aware ? 16 : 0), ldc = 32 + din;
    const uint32_t ha_n = a.head_aware ? 1u : 0u;
    uint32_t n_out;
    switch (seg) {
        case 0: n_out = 64 * (uint32_t)din; break;
        case 1: n_out = 64 * 64; break;
        case 2: n_out = 2 * 64; break;
        case 3: n_out = 32 * (uint32_t)ldc; break;
        case 4: n_out = 32 * 32; break;
        case 5: n_out = 4 * 32; break;
        case 6: n_out = (uint32_t)a.code_dim; break;
        case 7: n_out = ha_n * 16 * 4; break;
        case 8: n_out = ha_n * 32 * 16; break;
        case 9: n_out = ha_n * 16 * 32; break;
        case 10: n_out = ha_n * 16; break;
        case 11: n_out = ha_n * 32; break;
        default: n_out = ha_n * 16; break;
    }
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += gridDim.x * blockDim.x) {
        float v;
        switch (seg) {
            case 0: {
                const uint32_t n = i / din, k = i % din;
                v = k < 42 ? sum(TorsoSrPart::d0 + n * KD0 + k)
                    : (int)k < 42 + nh ? sum(TorsoSrPart::csd + n) * const_col(a, (int)k - 42)
                                       : sum(TorsoSrPart::d0 + n * KD0 + 42 + (k - 42 - nh));
                break;
            }
            case 1: v = sum(TorsoSrPart::d1 + i); break;
            case 2: v = sum(TorsoSrPart::d2 + i); break;
            case 3: {
                const uint32_t n = i / ldc, k = i % ldc;
                v = k < 74 ? sum(TorsoSrPart::c0 + n * KC0 + k)
                    : (int)k < 74 + nh ? sum(TorsoSrPart::csc + n) * const_col(a, (int)k - 74)
                                       : sum(TorsoSrPart::c0 + n * KC0 + 74 + (k - 74 - nh));
                break;
            }
            case 4: v = sum(TorsoSrPart::c1 + i); break;
            case 5: v = sum(TorsoSrPart::c2 + i); break;
            case 6: {
                v = 0.f;
                for (int n = 0; n < 64; ++n) v = fmaf(sum(TorsoSrPart::csd + n), a.w_def[0][n * din + 42 + i], v);
                for (int n = 0; n < 32; ++n) v = fmaf(sum(TorsoSrPart::csc + n), a.w_can[0][n * ldc + 74 + i], v);
                break;
            }
            case 7: v = sum(TorsoSrPart::hw0 + i); break;
            case 8: v = sum(TorsoSrPart::hw1 + i); break;
            case 9: v = sum(TorsoSrPart::hw2 + i); break;
            case 10: v = sum(TorsoSrPart::hb0 + i); break;
            case 11: v = sum(TorsoSrPart::hb1 + i); break;
            default: v = sum(TorsoSrPart::hb2 + i); break;
        }
        if (seg < 3) a.g_def[seg][i] = v;
        else if (seg < 6) a.g_can[seg - 3][i] = v;
        else if (seg == 6) a.g_code[i] = v;
        else if (seg < 10) a.g_ha_w[seg - 7][i] = v;
        else a.g_ha_b[seg - 10][i] = v;
    }
}

cudaError_t launch_torso_sr_field_relayout(const TorsoSrTrainArgs &a, cudaStream_t st) {
    k_torso_sr_field_relayout<<<grid_for(TorsoSrWt::total, 256), 256, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_torso_sr_field_bwd(const TorsoSrTrainArgs &a, cudaStream_t st) {
    static_assert(sizeof(Smem) <= 227 * 1024, "torso-SR training backward exceeds the per-CTA shared memory limit");
    cudaError_t e = cudaFuncSetAttribute(k_torso_sr_field_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    k_torso_sr_field_bwd<<<a.n_cta, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_torso_sr_field_reduce(const TorsoSrTrainArgs &a, cudaStream_t st) {
    k_torso_sr_field_reduce<<<dim3(32, 13), 256, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gfpp
