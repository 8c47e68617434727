// tc_pack.cu -- weight repacking for the wgmma path + a one-tile GEMM self-test of the wgmma plumbing.
#include "launch.cuh"
#include "ops.cuh"
#include "tc.cuh"

namespace gfpp {

using namespace tc;

// One K-tile of nn.Linear weights W[.][ld] (fp32) -> 16-bit hi (and lo) tiles in the GMMA K-major layout, ready to be
// bulk-copied into shared memory: tile row dst_row0+n, column k  <-  W[row0+n][col0+k] for n < N, k < kc.
// The destination must be zero-initialised (padding rows / columns stay zero).
__global__ void k_pack_tc_tile(const float *__restrict__ W, int ld, int row0, int col0, int N, int kc, int dst_row0,
                               int k16, int bf16, unsigned char *__restrict__ hi, unsigned char *__restrict__ lo) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N * kc; i += gridDim.x * blockDim.x) {
        const int n0 = i / kc, k = i - n0 * kc, n = dst_row0 + n0;
        const float v = W[(size_t)(row0 + n0) * ld + col0 + k];
        const uint32_t off = (k16 ? k16_off(n, k >> 3) : sw128_off(n, k >> 3)) + (uint32_t)(k & 7) * 2u;
        if (bf16) {
            const __nv_bfloat16 h = __float2bfloat16_rn(v);
            *reinterpret_cast<__nv_bfloat16 *>(hi + off) = h;
            if (lo) *reinterpret_cast<__nv_bfloat16 *>(lo + off) = __float2bfloat16_rn(v - __bfloat162float(h));
        } else {
            const __half h = __float2half_rn(v);
            *reinterpret_cast<__half *>(hi + off) = h;
            if (lo) *reinterpret_cast<__half *>(lo + off) = __float2half_rn(v - __half2float(h));
        }
    }
}

cudaError_t launch_pack_tc_tile(const float *W, int ld, int row0, int col0, int N, int kc, int dst_row0, int k16, int bf16,
                                unsigned char *hi, unsigned char *lo, cudaStream_t st) {
    const int total = N * kc;
    k_pack_tc_tile<<<grid_for((uint64_t)total, 256), 256, 0, st>>>(W, ld, row0, col0, N, kc, dst_row0, k16, bf16, hi, lo);
    return cudaGetLastError();
}

// The geo part of sigma L2 folded into color L0 (k_head_v2): W_fold[n][k] = sum_j Wc[n][c0 + j] * Ws[1 + j][k], n, j, k < 128
// (Wc: color L0 [.][ldc], its geo columns from c0; Ws: sigma L2 [129][128], row 0 = the sigma row).  Accumulated in double in
// ascending j, rounded to fp32 and then to fp16, and written as the two K = 64 SW128 tiles k_pack_tc_tile would make of it
// (tile k / 64 at tiles + (k / 64) * tile_bytes).
__global__ void k_pack_fold_tile(const float *__restrict__ Wc, int ldc, int c0, const float *__restrict__ Ws,
                                 unsigned char *__restrict__ tiles, int tile_bytes) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 128 * 128) return;
    const int n = i >> 7, k = i & 127;
    double acc = 0.0;
    for (int j = 0; j < 128; ++j) acc += (double)Wc[(size_t)n * ldc + c0 + j] * (double)Ws[(size_t)(1 + j) * 128 + k];
    const uint32_t off = (uint32_t)(k >> 6) * (uint32_t)tile_bytes + sw128_off(n, (k & 63) >> 3) + (uint32_t)(k & 7) * 2u;
    *reinterpret_cast<__half *>(tiles + off) = __float2half_rn((float)acc);
}

cudaError_t launch_pack_fold_tile(const float *Wc, int ldc, int c0, const float *Ws, unsigned char *tiles, int tile_bytes, cudaStream_t st) {
    k_pack_fold_tile<<<128 * 128 / 256, 256, 0, st>>>(Wc, ldc, c0, Ws, tiles, tile_bytes);
    return cudaGetLastError();
}

// A narrow layer W[N][ld] (N <= 8 outputs, K = 128 inputs, fp32) as the B operand of eight chained mma.sync m16n8k16, one per
// 16-wide k-block kb: lane l = 4n + t holds, for kb, the pair W[n][16kb + 2t .. +1] (b0) and W[n][16kb + 8 + 2t .. +1] (b1).
// Fragment word w = 2kb + (b1 ? 1 : 0) of lane l sits at (w / 4) * 512 + 16 l + 4 (w % 4): one conflict-free 16-byte load per lane
// gives two k-blocks.  Outputs n >= N are zero; every byte of the 2 KB image is written.  lo (when given) = rn16(W - rn16(W)).
__global__ void k_pack_narrow_b(const float *__restrict__ W, int ld, int N, unsigned char *__restrict__ hi, unsigned char *__restrict__ lo) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (n, k), n < 8, k < 128
    if (i >= 8 * 128) return;
    const int n = i >> 7, k = i & 127, kb = k >> 4, kk = k & 15;
    const int lane = 4 * n + ((kk & 7) >> 1), w = 2 * kb + (kk >> 3);
    const uint32_t off = (uint32_t)(w >> 2) * 512u + (uint32_t)lane * 16u + (uint32_t)(w & 3) * 4u + (uint32_t)(kk & 1) * 2u;
    const float v = n < N ? W[(size_t)n * ld + k] : 0.f;
    const __half h = __float2half_rn(v);
    *reinterpret_cast<__half *>(hi + off) = h;
    if (lo) *reinterpret_cast<__half *>(lo + off) = __float2half_rn(v - __half2float(h));
}

cudaError_t launch_pack_narrow_b(const float *W, int ld, int N, unsigned char *hi, unsigned char *lo, cudaStream_t st) {
    if (N < 1 || N > 8) return cudaErrorInvalidValue;
    k_pack_narrow_b<<<8 * 128 / 256, 256, 0, st>>>(W, ld, N, hi, lo);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// Self-test: out[128][N] = A[128][K] * W[N][K]^T through exactly the tile layouts, descriptors, wgmma issue and accumulator
// fragment layout the fused kernels use (warpgroup g computes rows 64g..64g+63).  K = 64*nt64 (+16 when k16_tail); the weight
// tiles come pre-packed.
struct TcTestSmem {
    unsigned char a_hi[3][16384];
    unsigned char a_lo[3][16384];
    unsigned char w_hi[3][18432];
    unsigned char w_lo[3][18432];
    unsigned long long bar_w;
};

template <int N, bool BF16, bool SPLIT>
__device__ __forceinline__ void selftest_mma(TcTestSmem &s, int K, int nt64, int k16_tail, float *__restrict__ out) {
    const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31, wwarp = (tid >> 5) & 3;
    const int ntiles = nt64 + (k16_tail ? 1 : 0);
    float d[N / 2];
    acc_zero(d);
    wg_fence();
    for (int t = 0; t < ntiles; ++t) {
        const bool is16 = k16_tail && t == nt64;
        // a partial last 64-wide tile only holds (K - 64*t)/16 k-steps of defined operand data
        const int k64 = K - (k16_tail ? 16 : 0);
        const int ks = is16 ? 1 : ((k64 - 64 * t) >= 64 ? 4 : (k64 - 64 * t) / 16);
        const uint32_t half = (uint32_t)wg * (is16 ? K16_HALF : SW128_HALF);
        const uint32_t a_hi = smem_u32(s.a_hi[t]) + half, a_lo = smem_u32(s.a_lo[t]) + half;
        const uint32_t w_hi = smem_u32(s.w_hi[t]), w_lo = smem_u32(s.w_lo[t]);
        for (int k = 0; k < ks; ++k) {
            const uint32_t adv = (uint32_t)k * 32u;   // 16 elements x 2 B inside the 128-byte swizzle row
            const uint64_t ah = is16 ? desc_k16(a_hi) : desc_sw128(a_hi + adv), wh = is16 ? desc_k16(w_hi) : desc_sw128(w_hi + adv);
            const uint32_t acc0 = (t > 0 || k > 0) ? 1u : 0u;
            if (SPLIT) {
                const uint64_t al = is16 ? desc_k16(a_lo) : desc_sw128(a_lo + adv), wl = is16 ? desc_k16(w_lo) : desc_sw128(w_lo + adv);
                wgmma<N, BF16>(d, al, wh, acc0);   // small terms first
                wgmma<N, BF16>(d, ah, wl, 1u);
                wgmma<N, BF16>(d, ah, wh, 1u);
            } else {
                wgmma<N, BF16>(d, ah, wh, acc0);
            }
        }
    }
    wg_commit();
    wg_wait<0>();
    acc_fence(d);
#pragma unroll
    for (int i = 0; i < N / 2; ++i) out[(size_t)(64 * wg + frag_row(i, lane, wwarp)) * N + frag_col(i, lane)] = d[i];
}

template <bool BF16, bool SPLIT>
__global__ void __launch_bounds__(256, 1) k_tc_selftest(const float *__restrict__ A, int K, const unsigned char *__restrict__ wt_hi,
                                                        const unsigned char *__restrict__ wt_lo, int N, int nt64, int k16_tail,
                                                        float *__restrict__ out) {
    extern __shared__ __align__(1024) unsigned char raw_[];
    unsigned char *raw = raw_ + ((1024u - (smem_u32(raw_) & 1023u)) & 1023u);  // SW128 tiles need 1024-byte alignment
    TcTestSmem &s = *reinterpret_cast<TcTestSmem *>(raw);
    const int tid = threadIdx.x;
    const int ntiles = nt64 + (k16_tail ? 1 : 0);
    if (tid == 32) {
        mbar_init(&s.bar_w, 1);
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t tile_bytes = 18432;
    if (tid == 0) {
        uint32_t bytes = 0;
        for (int t = 0; t < ntiles; ++t) bytes += tile_bytes * (SPLIT ? 2 : 1);
        mbar_expect_tx(&s.bar_w, bytes);
        for (int t = 0; t < ntiles; ++t) {
            bulk_g2s(s.w_hi[t], wt_hi + (size_t)t * tile_bytes, tile_bytes, &s.bar_w);
            if (SPLIT) bulk_g2s(s.w_lo[t], wt_lo + (size_t)t * tile_bytes, tile_bytes, &s.bar_w);
        }
    }
    // A: fp32 global -> 16-bit swizzled tiles; thread (row, part) converts chunks part, part+2, ...
    {
        const int row = tid & 127, part = tid >> 7;
        for (int c = part; c < K / 8; c += 2) {
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = A[(size_t)row * K + c * 8 + i];
            const int t = c / 8, cc = c % 8;
            const bool is16 = k16_tail && t == nt64;
            const uint32_t off = is16 ? k16_off(row, cc) : sw128_off(row, cc);
            store_chunk<BF16, SPLIT>(s.a_hi[t], s.a_lo[t], off, v);
        }
    }
    fence_async_smem();
    __syncthreads();
    mbar_wait(&s.bar_w, 0);
    if (N == 16) selftest_mma<16, BF16, SPLIT>(s, K, nt64, k16_tail, out);
    else if (N == 128) selftest_mma<128, BF16, SPLIT>(s, K, nt64, k16_tail, out);
    else selftest_mma<144, BF16, SPLIT>(s, K, nt64, k16_tail, out);
}

cudaError_t launch_tc_selftest(const float *A, int K, const unsigned char *wt_hi, const unsigned char *wt_lo, int N, int nt64,
                               int k16_tail, int precision, float *out, cudaStream_t st) {
    if (N != 16 && N != 128 && N != 144) return cudaErrorInvalidValue;   // the MMA widths the kernels use
    const size_t smem = sizeof(TcTestSmem) + 1024;
    cudaError_t e;
#define GO(BF, SP)                                                                                                     \
    e = cudaFuncSetAttribute(k_tc_selftest<BF, SP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);           \
    if (e != cudaSuccess) return e;                                                                                    \
    k_tc_selftest<BF, SP><<<1, 256, smem, st>>>(A, K, wt_hi, wt_lo, N, nt64, k16_tail, out);
    if (precision == FP16_X1) { GO(false, false) }
    else if (precision == BF16_X1) { GO(true, false) }
    else if (precision == BF16_X3) { GO(true, true) }
    else return cudaErrorInvalidValue;
#undef GO
    return cudaGetLastError();
}

}  // namespace gfpp
