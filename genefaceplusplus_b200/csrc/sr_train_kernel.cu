// sr_train_kernel.cu -- backward of the super-resolution head (sr_kernel.cu) on sm_90a, for the SR tasks' losses.
//
// Gradients are fp32 between layers.  The three tensor-core layers run their dgrad and wgrad products on TF32 wgmma with fp32
// accumulation: the non-gradient operand of every product is a value the forward already rounded to fp16 (the packed weights,
// the stored activations x0a, x0b, x1a, x1b), exact in tf32, so the one new rounding of the GEMMs is the gradient operand's
// round-to-nearest-even to tf32 (rn_tf32 below).  The toRGB stages differ from the forward in one more way: the forward's toRGB
// took the fp32 activation before its fp16 store, the backward rebuilds toRGB's output (for its clamp mask) and forms the toRGB
// weight gradients from the stored fp16 activation.  fp16 gradients are no option: a mean-reduced loss over a 512^2 x 3 image
// puts per-pixel gradients near fp16's subnormal range.
//
//   k_srb_rgb<64>     output stage at 2R: toRGB1's adjoint (3 -> 64) of the upstream image gradient times y'(x1b)
//   k_srb_rgb<128>    at R: adjoint of the 4-tap up-sampled skip -> g_img0, masked by toRGB0's clamp -> g_r0
//   k_srb_dgrad<0>    block1.conv1 (64 -> 64 at 2R), times y'(x1a)
//   k_srb_dgrad<1>    block1.conv0: the four output phases back to the R grid (K = 9 x 256), + toRGB0's adjoint, times y'(x0b)
//   k_srb_dgrad<2>    block0.conv1 (128 -> 128), times y'(x0a)
//   k_srb_in_dgrad    block0.conv0 (128 -> 3) on CUDA cores, + g_img0 (block 0's identity skip)
//   k_srb_wgrad<L>    the three GEMM weights, k_srb_in_wgrad the 27 x 128 input layer, k_srb_chan_sums biases and noise
//                     strengths, k_srb_rgb the toRGB weights and biases: per-CTA partials over a fixed slicing of the pixels,
//                     summed in ascending slice order by k_srb_sum -- no float atomics, repeated calls are bit-identical.
//
// dgrad is the forward's implicit GEMM (a tile = 128 pixels of one image row, K = 9 taps x channels in chunks of 64) on the
// gradient with flipped, transposed weights; the weight chunks stream through a 2-deep cp.async.bulk + mbarrier ring.  The A
// operand (the gradient) goes to wgmma from registers, the one place tf32 operands may come from.
// The derivative of lrelu_clamp is taken from the stored activation y, as the reference's bias_act backward does (ref = 'y'):
// sqrt(2) for y > 0, 0.2 sqrt(2) otherwise, 0 where |y| >= 256.
#include <math.h>

#include "launch.cuh"
#include "sr_kernel.cuh"
#include "sr_train_kernel.cuh"
#include "tc.cuh"

namespace gfpp {

using namespace tc;

namespace {

constexpr float kSqrt2 = 1.4142135623730951f;

__device__ __forceinline__ float dact(float y) { return fabsf(y) < 256.f ? (y > 0.f ? kSqrt2 : 0.2f * kSqrt2) : 0.f; }

// fp32 -> tf32 bit pattern, round to nearest even
__device__ __forceinline__ uint32_t rn_tf32(float x) {
    uint32_t r;
    asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ unsigned char *align1024(unsigned char *p) {
    return p + ((1024u - (smem_u32(p) & 1023u)) & 1023u);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// dgrad weight image of mode m: B[n][k], k = tap' * CG + c, holds the forward matrix entry W[c][(8 - tap') * N + n] (the tap
// flipped: the adjoint of a shift by +d is a shift by -d), read from the fp16 SW128 tiles of gfpp_sr_pack, as tf32 K8 blocks:
// chunk q = k / 64 of N x 256 bytes, k-step j inside it at j * N * 32, element at k16_off(n, (k & 7) / 4) + 4 (k & 3)
struct SrPackDgradArgs {
    const unsigned char *tiles[3];
    unsigned char *dst[3];
};
__global__ void k_srb_pack_dgrad(const __grid_constant__ SrPackDgradArgs a) {
    const int mode = blockIdx.y;
    const int CG = sr_dgrad_cg(mode), N = sr_dgrad_n(mode), l = sr_dgrad_fwd_layer(mode);
    const int NBf = sr_layer_nb(l), NRf = sr_layer_nrows(l);
    const int total = 9 * CG * N;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int n = i % N, k = i / N;
        const int tap = k / CG, c = k % CG;
        const int kf = (8 - tap) * N + n, cf = kf >> 6, kkf = kf & 63, nb = c / NRf, r = c % NRf;
        const size_t src = ((size_t)cf * NBf + nb) * NRf * 128 + sw128_off(r, kkf >> 3) + (uint32_t)(kkf & 7) * 2u;
        const float v = __half2float(*reinterpret_cast<const __half *>(a.tiles[l] + src));
        const int q = k >> 6, kk = k & 63;
        const size_t dst = (size_t)q * N * 256 + (size_t)(kk >> 3) * N * 32 + k16_off(n, (kk & 7) >> 2) + 4u * (uint32_t)(kk & 3);
        *reinterpret_cast<float *>(a.dst[mode] + dst) = v;
    }
}

cudaError_t launch_sr_pack_dgrad(const unsigned char *const tiles[3], unsigned char *const dst[3], cudaStream_t st) {
    SrPackDgradArgs a;
    for (int i = 0; i < 3; ++i) { a.tiles[i] = tiles[i]; a.dst[i] = dst[i]; }
    k_srb_pack_dgrad<<<dim3(144, 3), 256, 0, st>>>(a);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(256, 2) k_srb_dgrad(const __grid_constant__ SrDgradArgs a) {
    constexpr int CG = sr_dgrad_cg(MODE), N = sr_dgrad_n(MODE), CB = CG / 64, NC = 9 * CB, NB = N / 64;
    constexpr uint32_t CHUNK = (uint32_t)N * 256u;
    extern __shared__ __align__(1024) unsigned char smem_raw_[];
    unsigned char *w = align1024(smem_raw_);
    unsigned long long *bar = reinterpret_cast<unsigned long long *>(w + 2 * CHUNK);
    float *s_rgbw = reinterpret_cast<float *>(bar + 2);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7, wwarp = warp & 3;

    const int tiles_per_row = a.W / SR_TILE_ROWS;
    const int n_tiles = a.F * a.H * tiles_per_row;
    const int n_my = (int)blockIdx.x < n_tiles ? (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const uint32_t g_total = (uint32_t)n_my * (uint32_t)NC;

    if (tid == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        mbar_fence_init();
    }
    if (MODE == 1)
        for (int i = tid; i < 3 * N; i += 256) s_rgbw[i] = a.rgb_w[i];
    __syncthreads();
    if (tid == 0)
        for (uint32_t q = 0; q < 2 && q < g_total; ++q) {
            mbar_expect_tx(&bar[q], CHUNK);
            bulk_g2s(w + q * CHUNK, a.wt + (size_t)(q % NC) * CHUNK, CHUNK, &bar[q]);
        }

    uint32_t g = 0;
#pragma unroll 1
    for (int it = 0; it < n_my; ++it) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        const int xseg = tile % tiles_per_row, fy = tile / tiles_per_row;
        const int y = fy % a.H, f = fy / a.H, x0 = xseg * SR_TILE_ROWS;
        const int r0 = 64 * wg + 16 * wwarp + (lane >> 2);

        float d[NB][32];
#pragma unroll 1
        for (int c = 0; c < NC; ++c, ++g) {
            const uint32_t slot = g & 1u;
            const int tap = c / CB, cb = c - tap * CB;
            const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1, yy = y + dy;
            // A fragments of the chunk: rows r0 (a0, a2) and r0 + 8 (a1, a3), channels 8j + lane%4 (a0, a1) and + 4 (a2, a3)
            uint32_t av[8][4];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int xx = x0 + r0 + 8 * h + dx;
                const bool ok = (unsigned)yy < (unsigned)a.H && (unsigned)xx < (unsigned)a.W;
                const float *src;
                if (MODE == 1)   // phase cb = py * 2 + px of input pixel (yy, xx): the 2R pixel (2yy + py, 2xx + px)
                    src = a.g + (((size_t)f * 2 * a.H + 2 * (ok ? yy : 0) + (cb >> 1)) * 2 * a.W + 2 * (ok ? xx : 0) + (cb & 1)) * 64;
                else
                    src = a.g + (((size_t)f * a.H + (ok ? yy : 0)) * a.W + (ok ? xx : 0)) * CG + cb * 64;
#pragma unroll
                for (int j = 0; j < 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) av[j][2 * e + h] = rn_tf32(ok ? __ldg(src + 8 * j + (lane & 3) + 4 * e) : 0.f);
            }
            mbar_wait(&bar[slot], (g >> 1) & 1u);
            const uint32_t base = smem_u32(w + slot * CHUNK);
            wg_fence();
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int nb = 0; nb < NB; ++nb)
                    wgmma_tf32<64>(d[nb], av[j], desc_tf32_k8(base + (uint32_t)(j * N * 32 + nb * 2048)), (c > 0 || j > 0) ? 1u : 0u);
            wg_commit();
            wg_wait<0>();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) acc_fence(d[nb]);
            __syncthreads();   // both warpgroups are done with this slot
            if (tid == 0 && g + 2 < g_total) {
                const uint32_t q = g + 2;
                mbar_expect_tx(&bar[slot], CHUNK);
                bulk_g2s(w + slot * CHUNK, a.wt + (size_t)(q % NC) * CHUNK, CHUNK, &bar[slot]);
            }
        }

#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int row = 64 * wg + frag_row(i, lane, wwarp), col = nb * 64 + frag_col(i, lane);
                const size_t pix = ((size_t)f * a.H + y) * a.W + x0 + row;
                float v0 = d[nb][i], v1 = d[nb][i + 1];
                if (MODE == 1) {
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        const float gr = __ldg(a.g_rgb + pix * 3 + o);
                        v0 = fmaf(s_rgbw[o * N + col], gr, v0);
                        v1 = fmaf(s_rgbw[o * N + col + 1], gr, v1);
                    }
                }
                const __half2 y2 = *reinterpret_cast<const __half2 *>(a.act + pix * N + col);
                *reinterpret_cast<float2 *>(a.out + pix * N + col) = make_float2(v0 * dact(__low2float(y2)), v1 * dact(__high2float(y2)));
            }
        }
    }
}

template <int MODE>
static cudaError_t launch_sr_dgrad_t(const SrDgradArgs &a, cudaStream_t st) {
    const size_t smem = 1024 + 2 * (size_t)sr_dgrad_n(MODE) * 256 + 16 + 3 * 128 * 4;
    cudaError_t e = cudaFuncSetAttribute(k_srb_dgrad<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int n_tiles = a.F * a.H * (a.W / SR_TILE_ROWS);
    int blocks = sm_count() * 2;
    if (blocks > n_tiles) blocks = n_tiles;
    k_srb_dgrad<MODE><<<blocks, 256, smem, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sr_dgrad(int mode, const SrDgradArgs &a, cudaStream_t st) {
    if (a.W % SR_TILE_ROWS || a.F <= 0 || a.H <= 0) return cudaErrorInvalidValue;
    if (mode == 0) return launch_sr_dgrad_t<0>(a, st);
    if (mode == 1) return launch_sr_dgrad_t<1>(a, st);
    if (mode == 2) return launch_sr_dgrad_t<2>(a, st);
    return cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------------------------
// one CTA = one warpgroup = one (tap, 64 rows m, 64 channels ci) block of the weight gradient over one slice of the pixel tiles.
// K = the 128 pixels of a tile: A[m][k] = g[pixel k][m] from registers, B[ci][k] = x[pixel k + tap][ci] (fp16, exact in tf32)
// staged in shared memory as K8 blocks of 64 rows
template <int MODE>
__global__ void __launch_bounds__(128) k_srb_wgrad(const __grid_constant__ SrWgradArgs a) {
    constexpr int M = sr_wgrad_m(MODE), CI = sr_wgrad_ci(MODE), MB = M / 64, CIB = CI / 64;
    __shared__ __align__(1024) unsigned char sb[16 * 64 * 32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int item = blockIdx.x, tap = item / (MB * CIB), mb = (item / CIB) % MB, cib = item % CIB;
    const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1;
    const int s = blockIdx.y;
    const int tiles_per_row = a.W / SR_TILE_ROWS;
    const long long n_tiles = (long long)a.F * a.H * tiles_per_row;
    const long long t0 = n_tiles * s / a.slices, t1 = n_tiles * (s + 1) / a.slices;
    const int m0 = 16 * warp + (lane >> 2);

    float d[32];
    acc_zero(d);
#pragma unroll 1
    for (long long t = t0; t < t1; ++t) {
        const int xseg = (int)(t % tiles_per_row);
        const long long fy = t / tiles_per_row;
        const int y = (int)(fy % a.H), f = (int)(fy / a.H), x0 = xseg * SR_TILE_ROWS;
        __syncthreads();   // the previous tile's MMAs have finished reading sb (waited below)
        {
            const int yy = y + dy;
#pragma unroll 2
            for (int q = tid; q < SR_TILE_ROWS * 8; q += 128) {
                const int r = q >> 3, c8 = q & 7, xx = x0 + r + dx;
                uint4 v = make_uint4(0u, 0u, 0u, 0u);
                if ((unsigned)yy < (unsigned)a.H && (unsigned)xx < (unsigned)a.W)
                    v = __ldg(reinterpret_cast<const uint4 *>(a.x + (((size_t)f * a.H + yy) * a.W + xx) * CI + cib * 64) + c8);
                const __half *hv = reinterpret_cast<const __half *>(&v);
                const uint32_t kb = (uint32_t)(r >> 3) * 64u * 32u + 4u * (uint32_t)(r & 3);
#pragma unroll
                for (int e = 0; e < 8; ++e)
                    *reinterpret_cast<float *>(sb + kb + k16_off(c8 * 8 + e, (r & 7) >> 2)) = __half2float(hv[e]);
            }
        }
        uint32_t av[16][4];
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int px = x0 + 8 * j + (lane & 3) + 4 * e;
                const float *src;
                if (MODE == 1)
                    src = a.g + (((size_t)f * 2 * a.H + 2 * y + (mb >> 1)) * 2 * a.W + 2 * px + (mb & 1)) * 64;
                else
                    src = a.g + (((size_t)f * a.H + y) * a.W + px) * M + mb * 64;
#pragma unroll
                for (int h = 0; h < 2; ++h) av[j][2 * e + h] = rn_tf32(__ldg(src + m0 + 8 * h));
            }
        fence_async_smem();
        __syncthreads();
        const uint32_t base = smem_u32(sb);
        wg_fence();
#pragma unroll
        for (int j = 0; j < 16; ++j) wgmma_tf32<64>(d, av[j], desc_tf32_k8(base + (uint32_t)(j * 64 * 32)), 1u);
        wg_commit();
        wg_wait<0>();
        acc_fence(d);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
        const int m = mb * 64 + frag_row(i, lane, warp), n = cib * 64 + frag_col(i, lane);
        a.partial[((size_t)s * M + m) * (9 * CI) + tap * CI + n] = d[i];
    }
}

cudaError_t launch_sr_wgrad(int mode, const SrWgradArgs &a, cudaStream_t st) {
    if (a.W % SR_TILE_ROWS || a.F <= 0 || a.H <= 0 || a.slices <= 0) return cudaErrorInvalidValue;
    if (mode == 0) k_srb_wgrad<0><<<dim3(9 * 1 * 1, a.slices), 128, 0, st>>>(a);
    else if (mode == 1) k_srb_wgrad<1><<<dim3(9 * 4 * 2, a.slices), 128, 0, st>>>(a);
    else if (mode == 2) k_srb_wgrad<2><<<dim3(9 * 2 * 2, a.slices), 128, 0, st>>>(a);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// toRGB stages, one thread per pixel of a 128-pixel row segment, SR_SIMT_SLICES CTAs striding over the segments.
//   C = 64  (2R grid):  r = toRGB1(x1b); g_r = g * [|r| < 256]; g_pre[c] = sum_o rgb_w[o][c] g_r[o] * y'(x1b[c])
//   C = 128 (R grid):   g_img0 = adjoint of the up-sampled skip of g; r = toRGB0(x0b); g_r0 = g_img0 * [|r| < 256]
// rgb_part: per CTA sum_p g_r[o] x[c] ([3][C], o-major) and sum_p g_r[o] (3)
template <int C>
__global__ void __launch_bounds__(128) k_srb_rgb(const float *__restrict__ g, const __half *__restrict__ x, const float *__restrict__ rgb_w,
                                                 const float *__restrict__ rgb_b, int F, int H, float *__restrict__ g_pre,
                                                 float *__restrict__ g_img0, float *__restrict__ g_r0, float *__restrict__ rgb_part) {
    constexpr int NP = 3 * C + 3;
    __shared__ float s_w[3 * C];
    __shared__ float s_g[3][128];
    __shared__ __align__(16) __half s_x[128][C + 8];   // 16-byte rows
    const int tid = threadIdx.x;
    for (int i = tid; i < 3 * C; i += 128) s_w[i] = rgb_w[i];
    __syncthreads();
    const int W = H, tiles_per_row = W / 128;
    const long long n_tiles = (long long)F * H * tiles_per_row;
    float acc[(NP + 127) / 128];
#pragma unroll
    for (int k = 0; k < (NP + 127) / 128; ++k) acc[k] = 0.f;
    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int xseg = (int)(t % tiles_per_row);
        const long long fy = t / tiles_per_row;
        const int y = (int)(fy % H), f = (int)(fy / H), xp = xseg * 128 + tid;
        const size_t pix = ((size_t)f * H + y) * W + xp;
        float xv[C];
#pragma unroll
        for (int q = 0; q < C / 8; ++q) {
            const uint4 u = __ldg(reinterpret_cast<const uint4 *>(x + pix * C) + q);
            const __half *hv = reinterpret_cast<const __half *>(&u);
#pragma unroll
            for (int e = 0; e < 8; ++e) xv[8 * q + e] = __half2float(hv[e]);
            if (rgb_part) *reinterpret_cast<uint4 *>(&s_x[tid][8 * q]) = u;
        }
        float gin[3];
        if (C == 64) {
#pragma unroll
            for (int o = 0; o < 3; ++o) gin[o] = __ldg(g + (((size_t)f * 3 + o) * H + y) * W + xp);
        } else {   // adjoint of upsampled_skip: per axis, low-res i takes 0.75 from 2i and 2i+1 and 0.25 from 2i-1 and 2i+2
            const int H2 = 2 * H;
            gin[0] = gin[1] = gin[2] = 0.f;
#pragma unroll
            for (int jy = 0; jy < 4; ++jy) {
                const int Y = 2 * y - 1 + jy;
                if ((unsigned)Y >= (unsigned)H2) continue;
                const float wy = (jy == 1 || jy == 2) ? 0.75f : 0.25f;
#pragma unroll
                for (int jx = 0; jx < 4; ++jx) {
                    const int X = 2 * xp - 1 + jx;
                    if ((unsigned)X >= (unsigned)H2) continue;
                    const float wgt = wy * ((jx == 1 || jx == 2) ? 0.75f : 0.25f);
#pragma unroll
                    for (int o = 0; o < 3; ++o) gin[o] = fmaf(wgt, __ldg(g + (((size_t)f * 3 + o) * H2 + Y) * H2 + X), gin[o]);
                }
            }
#pragma unroll
            for (int o = 0; o < 3; ++o) g_img0[pix * 3 + o] = gin[o];
        }
        float gr[3];
#pragma unroll
        for (int o = 0; o < 3; ++o) {
            float r = __ldg(rgb_b + o);
#pragma unroll
            for (int c = 0; c < C; ++c) r = fmaf(s_w[o * C + c], xv[c], r);
            gr[o] = fabsf(r) < 256.f ? gin[o] : 0.f;
        }
        if (C == 64) {
#pragma unroll
            for (int q = 0; q < C / 4; ++q) {
                float v[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = 4 * q + e;
                    v[e] = fmaf(s_w[2 * C + c], gr[2], fmaf(s_w[C + c], gr[1], s_w[c] * gr[0])) * dact(xv[c]);
                }
                reinterpret_cast<float4 *>(g_pre + pix * C)[q] = make_float4(v[0], v[1], v[2], v[3]);
            }
        } else {
#pragma unroll
            for (int o = 0; o < 3; ++o) g_r0[pix * 3 + o] = gr[o];
        }
        if (rgb_part) {
#pragma unroll
            for (int o = 0; o < 3; ++o) s_g[o][tid] = gr[o];
            __syncthreads();
#pragma unroll
            for (int k = 0; k < (NP + 127) / 128; ++k) {
                const int i = tid + 128 * k;
                if (i < 3 * C) {
                    const int o = i / C, c = i % C;
                    float s = 0.f;
                    for (int p = 0; p < 128; ++p) s = fmaf(s_g[o][p], __half2float(s_x[p][c]), s);
                    acc[k] += s;
                } else if (i < NP) {
                    float s = 0.f;
                    for (int p = 0; p < 128; ++p) s += s_g[i - 3 * C][p];
                    acc[k] += s;
                }
            }
            __syncthreads();
        }
    }
    if (rgb_part) {
#pragma unroll
        for (int k = 0; k < (NP + 127) / 128; ++k) {
            const int i = tid + 128 * k;
            if (i < NP) rgb_part[(size_t)blockIdx.x * NP + i] = acc[k];
        }
    }
}

cudaError_t launch_sr_bwd_out(const float *g, const __half *x1b, const float *rgb_w, const float *rgb_b, int F, int R2, float *g_pre,
                              float *rgb_part, cudaStream_t st) {
    if (R2 % 128 || F <= 0) return cudaErrorInvalidValue;
    k_srb_rgb<64><<<SR_SIMT_SLICES, 128, 0, st>>>(g, x1b, rgb_w, rgb_b, F, R2, g_pre, nullptr, nullptr, rgb_part);
    return cudaGetLastError();
}

cudaError_t launch_sr_bwd_img0(const float *g, const __half *x0b, const float *rgb_w, const float *rgb_b, int F, int R, float *g_img0,
                               float *g_r0, float *rgb_part, cudaStream_t st) {
    if (R % 128 || F <= 0) return cudaErrorInvalidValue;
    k_srb_rgb<128><<<SR_SIMT_SLICES, 128, 0, st>>>(g, x0b, rgb_w, rgb_b, F, R, nullptr, g_img0, g_r0, rgb_part);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
// block0.conv0 (y[p][co] = sum_{tap, ci} w[tap * 3 + ci][co] x[p + tap][ci]): grad_in[q][ci] = g_img0[q][ci] +
// sum_{tap, co} w[tap * 3 + ci][co] g_pre[q - tap][co], one thread per pixel
__global__ void __launch_bounds__(256) k_srb_in_dgrad(const float *__restrict__ g_pre, const float *__restrict__ w,
                                                      const float *__restrict__ g_img0, int F, int R, float *__restrict__ grad_in) {
    __shared__ __align__(16) float sw[27 * 128];
    for (int i = threadIdx.x; i < 27 * 128; i += 256) sw[i] = w[i];
    __syncthreads();
    const long long n = (long long)F * R * R;
    for (long long q = blockIdx.x * 256ll + threadIdx.x; q < n; q += (long long)gridDim.x * 256) {
        const int x = (int)(q % R), y = (int)((q / R) % R);
        const long long f = q / ((long long)R * R);
        float acc[3] = {g_img0[q * 3], g_img0[q * 3 + 1], g_img0[q * 3 + 2]};
        for (int tap = 0; tap < 9; ++tap) {
            const int yy = y - (tap / 3 - 1), xx = x - (tap % 3 - 1);
            if ((unsigned)yy >= (unsigned)R || (unsigned)xx >= (unsigned)R) continue;
            const float4 *gp = reinterpret_cast<const float4 *>(g_pre + ((f * R + yy) * R + xx) * 128);
#pragma unroll 4
            for (int c4 = 0; c4 < 32; ++c4) {
                const float4 gv = __ldg(gp + c4);
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const float4 wv = reinterpret_cast<const float4 *>(sw + (tap * 3 + ci) * 128)[c4];
                    acc[ci] = fmaf(wv.w, gv.w, fmaf(wv.z, gv.z, fmaf(wv.y, gv.y, fmaf(wv.x, gv.x, acc[ci]))));
                }
            }
        }
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) grad_in[q * 3 + ci] = acc[ci];
    }
}

cudaError_t launch_sr_in_dgrad(const float *g_pre, const float *w, const float *g_img0, int F, int R, float *grad_in, cudaStream_t st) {
    k_srb_in_dgrad<<<grid_for((uint64_t)F * R * R, 256), 256, 0, st>>>(g_pre, w, g_img0, F, R, grad_in);
    return cudaGetLastError();
}

// partial[s][k][co] = sum over the pixels p of slice s of g_pre[p][co] x[p + tap][ci], k = tap * 3 + ci; thread = co
__global__ void __launch_bounds__(128) k_srb_in_wgrad(const float *__restrict__ g_pre, const float *__restrict__ x, int F, int R,
                                                      float *__restrict__ partial) {
    const int co = threadIdx.x, s = blockIdx.x;
    const long long n = (long long)F * R * R, p0 = n * s / gridDim.x, p1 = n * (s + 1) / gridDim.x;
    float acc[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) acc[k] = 0.f;
    for (long long p = p0; p < p1; ++p) {
        const int px = (int)(p % R), py = (int)((p / R) % R);
        const long long f = p / ((long long)R * R);
        const float gv = __ldg(g_pre + p * 128 + co);
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int yy = py + tap / 3 - 1, xx = px + tap % 3 - 1;
            if ((unsigned)yy >= (unsigned)R || (unsigned)xx >= (unsigned)R) continue;
            const float *xp = x + ((f * R + yy) * R + xx) * 3;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) acc[tap * 3 + ci] = fmaf(gv, __ldg(xp + ci), acc[tap * 3 + ci]);
        }
    }
#pragma unroll
    for (int k = 0; k < 27; ++k) partial[((size_t)s * 27 + k) * 128 + co] = acc[k];
}

cudaError_t launch_sr_in_wgrad(const float *g_pre, const float *x, int F, int R, float *partial, cudaStream_t st) {
    k_srb_in_wgrad<<<SR_SIMT_SLICES, 128, 0, st>>>(g_pre, x, F, R, partial);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256) k_srb_chan_sums(const float *__restrict__ g, int F, long long P, const float *__restrict__ raw,
                                                       int raw_per_frame, float *__restrict__ partial) {
    constexpr int G = 256 / C;
    __shared__ float s_sum[256], s_nd[256];
    const int tid = threadIdx.x, c = tid % C, sub = tid / C, s = blockIdx.x;
    const long long n = (long long)F * P, p0 = n * s / gridDim.x, p1 = n * (s + 1) / gridDim.x;
    float sum = 0.f, nd = 0.f;
    for (long long p = p0 + sub; p < p1; p += G) {
        const float v = __ldg(g + p * C + c);
        sum += v;
        if (raw) nd = fmaf(v, __ldg(raw + (raw_per_frame ? p : p % P)), nd);
    }
    s_sum[tid] = sum;
    s_nd[tid] = nd;
    __syncthreads();
    if (tid < C) {
        float t = 0.f;
        for (int k = 0; k < G; ++k) t += s_sum[k * C + tid];
        partial[(size_t)s * (C + 1) + tid] = t;
    }
    if (tid == 0) {
        float t = 0.f;
        for (int k = 0; k < 256; ++k) t += s_nd[k];
        partial[(size_t)s * (C + 1) + C] = t;
    }
}

cudaError_t launch_sr_chan_sums(const float *g, int C, int F, long long P, const float *raw, int raw_per_frame, float *partial,
                                cudaStream_t st) {
    if (C == 64) k_srb_chan_sums<64><<<SR_SIMT_SLICES, 256, 0, st>>>(g, F, P, raw, raw_per_frame, partial);
    else if (C == 128) k_srb_chan_sums<128><<<SR_SIMT_SLICES, 256, 0, st>>>(g, F, P, raw, raw_per_frame, partial);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

__global__ void k_srb_sum(const float *__restrict__ part, int S, int stride, int col0, int n, float *__restrict__ out) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float t = 0.f;
        for (int s = 0; s < S; ++s) t += part[(size_t)s * stride + col0 + i];
        out[i] = t;
    }
}

cudaError_t launch_sr_sum_cols(const float *part, int S, int stride, int col0, int n, float *out, cudaStream_t st) {
    k_srb_sum<<<grid_for((uint64_t)n, 256), 256, 0, st>>>(part, S, stride, col0, n, out);
    return cudaGetLastError();
}

}  // namespace gfpp
