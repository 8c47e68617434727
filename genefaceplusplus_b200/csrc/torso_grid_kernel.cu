// torso_grid_kernel.cu -- the torso fields at arbitrary points: forward_torso of the plain torso model (radnerf_torso.py:51-84)
// and of the torso-SR model (radnerf_torso_sr.py:73-113), for RADNeRFTorso.forward_torso and for the cell query of
// update_extra_state (radnerf_torso.py:201-242, radnerf_torso_sr.py:246-288).
//
// Same tiling and arithmetic as the render epilogues (k_epilogue, k_torso_sr), which stay separate kernels so that the render
// path is untouched: CTAs take tiles of 128 points, fp32 FFMA tile GEMMs out of shared memory, accurate sinf, the constant
// columns of the first layers (pose or jaw landmarks, and the code) folded by the frame-bias kernels with F = 1.  There is no
// occupancy mask: every point is evaluated.  The SR field's head-aware encoder sees image = weights_sum = 0, as the reference's
// refresh passes it; its 16 outputs are then the same for every point and are computed once per CTA.
#include "launch.cuh"
#include "torso_common.cuh"
#include "torso_grid_kernel.cuh"
#include "torso_sr_kernel.cuh"

namespace gfpp {

using namespace torsoc;

namespace {

constexpr int TP = 128;    // points per tile
constexpr int NT = 256;

template <bool SR> struct QShape;
// plain: deform input [enc_x 42 | pad 2], canonical input [tiled2D(x) 32 | enc_x 42 | pad 2]
template <> struct QShape<false> { static constexpr int KD0 = 44, KC0 = 76, LDT = 84; };
// SR: deform input [enc_x 42 | head-aware 16 | pad 2], canonical input [tiled2D(x) 32 | the same]
template <> struct QShape<true> { static constexpr int KD0 = TORSO_SR_KD0, KC0 = TORSO_SR_KC0, LDT = 100; };

template <bool SR> struct QSmem {
    static constexpr int KD0 = QShape<SR>::KD0, KC0 = QShape<SR>::KC0, LDT = QShape<SR>::LDT, LDE = KD0;
    float A[TP * LDT];
    float E[TP * LDE];
    float wd0[KD0 * 64], wd1[64 * 64], wc0[KC0 * 32], wc1[32 * 32];
    float wd2[2 * 64], wc2[4 * 32];
    float x2[2 * TP];
    float dxy[2 * TP];
    float h2[32], hae[16];
};

__device__ __forceinline__ float leaky002(float x) { return x > 0.f ? x : 0.02f * x; }

// point p in torso-grid coordinates [-1,1]^2: xy[p], or cell (p % H, p / H) jittered as radnerf_torso.py:221-227 does in fp32:
// xys = (2*c/(H-1) - 1) * (1 - 1/H) + (noise*2 - 1) * (1/H)
__device__ __forceinline__ void query_point(const TorsoQueryArgs &q, uint32_t p, float (&pos)[2]) {
    if (q.xy) { pos[0] = q.xy[2 * (size_t)p]; pos[1] = q.xy[2 * (size_t)p + 1]; return; }
    const uint32_t H = q.grid_size, c[2] = {p % H, p / H};
    const float *nz = q.noise + ((size_t)c[0] * H + c[1]) * 2;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const float xs = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, (float)c[k]), (float)(H - 1)), 1.0f);
        const float r = __fmul_rn(__fsub_rn(__fmul_rn(nz[k], 2.0f), 1.0f), q.hgs);
        pos[k] = __fadd_rn(__fmul_rn(xs, q.cell_scale), r);
    }
}

template <bool SR>
__device__ __forceinline__ void torso_query_body(const TorsoQueryArgs &q, unsigned char *smem_raw) {
    using S = QSmem<SR>;
    constexpr int KD0 = S::KD0, KC0 = S::KC0, LDT = S::LDT, LDE = S::LDE, HALF = KD0 / 2;
    S &s = *reinterpret_cast<S *>(smem_raw);
    const int tid = threadIdx.x;
    for (int i = tid; i < KD0 * 64; i += NT) s.wd0[i] = q.w_def0[i];
    for (int i = tid; i < 64 * 64; i += NT) s.wd1[i] = q.w_def1[i];
    for (int i = tid; i < KC0 * 32; i += NT) s.wc0[i] = q.w_can0[i];
    for (int i = tid; i < 32 * 32; i += NT) s.wc1[i] = q.w_can1[i];
    for (int i = tid; i < 2 * 64; i += NT) s.wd2[i] = q.w_def2[i];
    for (int i = tid; i < 4 * 32; i += NT) s.wc2[i] = q.w_can2[i];
    if (SR) {
        // head_color_weights_encoder(cat[0, 0]) in k_torso_sr's operation order: L0 of a zero input is its bias
        if (tid < 32) {
            float t = 0.f;
            if (q.ha) {
                t = q.ha[TORSO_SR_HA_B1 + tid];
                for (int k = 0; k < 16; ++k) t = fmaf(leaky002(q.ha[TORSO_SR_HA_B0 + k]), q.ha[TORSO_SR_HA_W1 + k * 32 + tid], t);
            }
            s.h2[tid] = leaky002(t);
        }
        __syncthreads();
        if (tid < 16) {
            float o = 0.f;
            if (q.ha) {
                o = q.ha[TORSO_SR_HA_B2 + tid];
                for (int k = 0; k < 32; ++k) o = fmaf(s.h2[k], q.ha[TORSO_SR_HA_W2 + k * 16 + tid], o);
            }
            s.hae[tid] = o;
        }
    }
    __syncthreads();
    const int ty = tid >> 4, tx = tid & 15;
    const int slot = tid & (TP - 1), lg = tid >> 7;
    const uint32_t n_tiles = (q.n + TP - 1) / TP;

    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t p = tile * TP + slot;
        const bool in_range = p < q.n;
        // ---- deform input: enc_x = freq10(shrink * x) [| head-aware encoding] | zero pad ----
        {
            float x[2] = {0.f, 0.f};
            if (in_range) {
                float pos[2];
                query_point(q, p, pos);
                x[0] = __fmul_rn(pos[0], q.torso_shrink); x[1] = __fmul_rn(pos[1], q.torso_shrink);
            }
            for (int c = lg * HALF; c < lg * HALF + HALF; ++c) {
                const float v = c < 42 ? freq_entry(x, 2, c) : (SR && c < 58) ? s.hae[c - 42] : 0.f;
                s.E[slot * LDE + c] = v;
                s.A[slot * LDT + c] = v;
            }
            if (lg == 0) { s.x2[slot] = x[0]; s.x2[TP + slot] = x[1]; }
        }
        __syncthreads();
        // ---- deform net -> 64 -> 64 -> 2 ----
        {
            float acc[8][4] = {};
            small_gemm<4, KD0, LDT>(acc, s.A, s.wd0, ty, tx);
            __syncthreads();
            store_relu<4, LDT>(acc, s.A, q.bias_def, ty, tx);
            __syncthreads();
        }
        {
            float acc[8][4] = {};
            small_gemm<4, 64, LDT>(acc, s.A, s.wd1, ty, tx);
            __syncthreads();
            store_relu<4, LDT>(acc, s.A, nullptr, ty, tx);
            __syncthreads();
        }
        {
            const int row = tid >> 1, half = tid & 1;
            float v0 = 0.f, v1 = 0.f;
            for (int k = half * 32; k < half * 32 + 32; ++k) {
                const float xk = s.A[row * LDT + k];
                v0 = fmaf(xk, s.wd2[k], v0);
                v1 = fmaf(xk, s.wd2[64 + k], v1);
            }
            v0 += __shfl_xor_sync(0xffffffffu, v0, 1);
            v1 += __shfl_xor_sync(0xffffffffu, v1, 1);
            if (half == 0) {
                s.dxy[row] = v0; s.dxy[TP + row] = v1;
                s.x2[row] = fminf(fmaxf(s.x2[row] + v0, -1.f), 1.f);           // x = (x + dx).clamp(-1, 1)
                s.x2[TP + row] = fminf(fmaxf(s.x2[TP + row] + v1, -1.f), 1.f);
            }
        }
        __syncthreads();
        // ---- canonical input: [tiled2D(x) 32 | deform input] ----
        {
            const float u = __fdiv_rn(__fadd_rn(s.x2[slot], 1.0f), 2.0f), v = __fdiv_rn(__fadd_rn(s.x2[TP + slot], 1.0f), 2.0f);
#pragma unroll 2
            for (int l = lg * 8; l < lg * 8 + 8; ++l)
                *reinterpret_cast<float2 *>(s.A + slot * LDT + 2 * l) = grid_lookup2(q.tor_gm, q.tor_tab, l, u, v);
            for (int c = lg * HALF; c < lg * HALF + HALF; ++c) s.A[slot * LDT + 32 + c] = s.E[slot * LDE + c];
        }
        __syncthreads();
        // ---- canonical net -> 32 -> 32 -> 4, sigmoid ----
        {
            float acc[8][2] = {};
            small_gemm<2, KC0, LDT>(acc, s.A, s.wc0, ty, tx);
            __syncthreads();
            store_relu<2, LDT>(acc, s.A, q.bias_can, ty, tx);
            __syncthreads();
        }
        {
            float acc[8][2] = {};
            small_gemm<2, 32, LDT>(acc, s.A, s.wc1, ty, tx);
            __syncthreads();
            store_relu<2, LDT>(acc, s.A, nullptr, ty, tx);
            __syncthreads();
        }
        {
            const int row = tid >> 1, half = tid & 1;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            for (int k = half * 16; k < half * 16 + 16; ++k) {
                const float xk = s.A[row * LDT + k];
#pragma unroll
                for (int o = 0; o < 4; ++o) v[o] = fmaf(xk, s.wc2[o * 32 + k], v[o]);
            }
#pragma unroll
            for (int o = 0; o < 4; ++o) v[o] += __shfl_xor_sync(0xffffffffu, v[o], 1);
            const uint32_t pr = tile * TP + row;
            if (half == 0 && pr < q.n) {
                q.alpha[pr] = 1.0f / (1.0f + expf(-v[0]));
                if (q.color) {
#pragma unroll
                    for (int o = 0; o < 3; ++o) q.color[3 * (size_t)pr + o] = 1.0f / (1.0f + expf(-v[1 + o]));
                }
                if (q.deform) { q.deform[2 * (size_t)pr] = s.dxy[row]; q.deform[2 * (size_t)pr + 1] = s.dxy[TP + row]; }
            }
        }
        __syncthreads();
    }
}

}  // namespace

__global__ void __launch_bounds__(256, 2) k_torso_query(const __grid_constant__ TorsoQueryArgs q) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    torso_query_body<false>(q, smem_raw);
}

__global__ void __launch_bounds__(256, 1) k_torso_sr_query(const __grid_constant__ TorsoQueryArgs q) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    torso_query_body<true>(q, smem_raw);
}

namespace {
template <bool SR>
cudaError_t launch_query(void (*kern)(TorsoQueryArgs), int ctas_per_sm, const TorsoQueryArgs &q, cudaStream_t st) {
    constexpr int bytes = (int)sizeof(QSmem<SR>);
    static_assert(sizeof(QSmem<SR>) <= 227 * 1024, "torso query exceeds the per-CTA shared memory limit");
    // function attributes are per device: set on every launch, never cached process-wide
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    const uint32_t tiles = (q.n + TP - 1) / TP;
    uint32_t blocks = (uint32_t)(ctas_per_sm * sm_count());
    if (tiles < blocks) blocks = tiles > 0 ? tiles : 1;
    kern<<<blocks, NT, bytes, st>>>(q);
    return cudaGetLastError();
}
}  // namespace

cudaError_t launch_torso_query(const TorsoQueryArgs &q, cudaStream_t st) { return launch_query<false>(k_torso_query, 2, q, st); }
cudaError_t launch_torso_sr_query(const TorsoQueryArgs &q, cudaStream_t st) { return launch_query<true>(k_torso_sr_query, 1, q, st); }

}  // namespace gfpp
