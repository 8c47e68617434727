// sr_kernel.cu -- super-resolution head of the SR checkpoints (256x256 NeRF image -> 512x512) on sm_90a.
//
// Replaces `Superresolution.forward` of modules/radnerfs/radnerf_sr.py:15-48, which the reference assembles from StyleGAN2
// synthesis blocks (modules/eg3ds/models/superresolution.py:159-257, networks_stylegan2.py:286-475) and runs as per-sample
// grouped cuDNN convolutions + upfirdn2d / bias_act custom ops.  The network always feeds the constant latent w = 1
// (radnerf_sr.py:33-34), so style modulation and demodulation are constants of the checkpoint: the host folds them into
// plain convolution weights once (genefaceplusplus_b200/superres.py) and the six layers become four launches per clip chunk:
//
//   k_sr_conv_in   block0.conv0    3 -> 128, 3x3          fp32 FFMA (K = 27 is no tensor-core shape), fp16 NHWC out
//   k_sr_conv<0>   block0.conv1  128 -> 128, 3x3          implicit GEMM on wgmma;   epilogue: noise, bias, leaky-ReLU*sqrt2,
//                                                         clamp, fp16 NHWC out + fused toRGB (128 -> 3, fp32) + rgb skip -> img0
//   k_sr_conv<1>   block1.conv0  128 -> 64, up x2         transposed stride-2 conv + [1,3,3,1] FIR merged into four 3x3 phase
//                                                         kernels on the INPUT grid: one GEMM with N = 4 x 64, no 513x513
//                                                         intermediate, no separate filter pass
//   k_sr_conv<2>   block1.conv1   64 -> 64, 3x3 at 512^2  implicit GEMM; epilogue: activation, fused toRGB, + the 2x FIR
//                                                         up-sampled img0 (closed form: 4 taps), optional clamp -> [F,3,512,512]
//                                                         and/or the uint8 video frames [F,512,512,3] (interleaved, as imageio
//                                                         takes them), each store optional
//
// Implicit GEMM: a tile is 128 consecutive pixels of one image row (the 128 rows of the MMA); K runs over the 9 taps x
// C_in in chunks of 64 channels.  For every chunk the CTA's threads copy the shifted 128 x 64 fp16 window of the NHWC
// activation straight into a GMMA K-major SW128 operand tile (one 16-byte load + one 16-byte store per thread and task,
// zeros outside the image), double-buffered against the MMAs (one wgmma group of each warpgroup stays in flight while the
// next window is copied); the weight chunks stream through a 4-deep cp.async.bulk + mbarrier ring; the two warpgroups of
// the CTA own pixel rows 0-63 and 64-127 and keep their accumulators (64 / 128 / 32 fp32 registers) for the epilogue.  Operands are fp16, accumulation fp32 -- the reference runs these blocks in fp16 on CUDA
// (use_fp16 of the synthesis blocks), toRGB and the skip path stay fp32.
#include <math.h>

#include "launch.cuh"
#include "sr_kernel.cuh"
#include "tc.cuh"

namespace gfpp {

using namespace tc;

namespace {

constexpr int TM = SR_TILE_ROWS;
constexpr int NT = 256;
constexpr int A_TILE = 16384;   // 128 rows x 64 k x 2 B (SW128)
constexpr int RING = 4;         // weight chunks in flight
constexpr float kSqrt2 = 1.4142135623730951f;

template <int LAYER>
struct SmemSR {
    alignas(1024) unsigned char a[2][A_TILE];
    alignas(1024) unsigned char w[RING][sr_layer_chunk_bytes(LAYER)];
    float bias[128];
    float rgbw[3 * 128];
    float part[3 * TM];
    unsigned long long bar_wfull[RING];
};

// bias_act of the synthesis layers: leaky-ReLU(0.2) * sqrt(2), then clamp to +-256 (networks_stylegan2.py:330-333)
__device__ __forceinline__ float lrelu_clamp(float t) {
    t = (t < 0.f ? 0.2f * t : t) * kSqrt2;
    return fminf(fmaxf(t, -256.f), 256.f);
}

// upfirdn2d.upsample2d with the [1,3,3,1] binomial filter at output pixel (y, x) of the 2h x 2w image: zero insertion,
// pad (2,1,2,1), filter * 4 -- per axis the even outputs are 0.25 * in[i-1] + 0.75 * in[i], the odd ones 0.75 * in[i] +
// 0.25 * in[i+1], with zeros outside the image
__device__ __forceinline__ void upsampled_skip(const float *__restrict__ img, int h, int w, int y, int x, float (&o)[3]) {
    const int yi = y >> 1, xi = x >> 1;
    const int y0 = (y & 1) ? yi : yi - 1, x0 = (x & 1) ? xi : xi - 1;
    const float wy0 = (y & 1) ? 0.75f : 0.25f, wx0 = (x & 1) ? 0.75f : 0.25f;
    o[0] = o[1] = o[2] = 0.f;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int yy = y0 + j;
        if ((unsigned)yy >= (unsigned)h) continue;
        const float wy = j == 0 ? wy0 : 1.0f - wy0;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int xx = x0 + i;
            if ((unsigned)xx >= (unsigned)w) continue;
            const float wgt = wy * (i == 0 ? wx0 : 1.0f - wx0);
            const float *p = img + ((size_t)yy * w + xx) * 3;
            o[0] = fmaf(wgt, __ldg(p), o[0]);
            o[1] = fmaf(wgt, __ldg(p + 1), o[1]);
            o[2] = fmaf(wgt, __ldg(p + 2), o[2]);
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
template <int LAYER>
__global__ void __launch_bounds__(NT, LAYER == 1 ? 1 : 2) k_sr_conv(const __grid_constant__ SrConvArgs a) {
    constexpr int CIN = sr_layer_cin(LAYER), CB = CIN / 64, NC = sr_layer_nchunk(LAYER);
    constexpr int NB = sr_layer_nb(LAYER), NROWS = sr_layer_nrows(LAYER);
    constexpr uint32_t WCHUNK = (uint32_t)sr_layer_chunk_bytes(LAYER);
    constexpr int COUT = LAYER == 0 ? 128 : 64;
    constexpr int R = NROWS / 2;   // accumulator registers per N-block

    extern __shared__ __align__(1024) unsigned char smem_raw_[];
    unsigned char *smem_raw = smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u);
    SmemSR<LAYER> &s = *reinterpret_cast<SmemSR<LAYER> *>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7, wwarp = warp & 3;

    const int tiles_per_row = a.W / TM;
    const int n_tiles = a.F * a.H * tiles_per_row;
    const int n_my = (int)blockIdx.x < n_tiles ? (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const uint32_t g_total = (uint32_t)n_my * (uint32_t)NC;

    // ---- one-time setup ----
    if (tid == 32) {
        for (int i = 0; i < RING; ++i) mbar_init(&s.bar_wfull[i], 1);
        mbar_fence_init();
    }
    for (int i = tid; i < COUT; i += NT) s.bias[i] = a.bias[i];
    if (LAYER != 1)
        for (int i = tid; i < 3 * COUT; i += NT) s.rgbw[i] = a.rgb_w[i];
    __syncthreads();
    if (warp == 0) {   // first RING weight chunks of the (cyclic) stream
        if (elect_one()) {
            for (uint32_t q = 0; q < (uint32_t)RING && q < g_total; ++q) {
                mbar_expect_tx(&s.bar_wfull[q], WCHUNK);
                bulk_g2s(s.w[q], a.wt + (size_t)(q % NC) * WCHUNK, WCHUNK, &s.bar_wfull[q]);
            }
        }
        __syncwarp();
    }

    uint32_t g = 0;                                                 // running K-chunk counter (CTA-uniform)
#pragma unroll 1
    for (int it = 0; it < n_my; ++it) {
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        const int xseg = tile % tiles_per_row;
        const int fy = tile / tiles_per_row;
        const int y = fy % a.H, f = fy / a.H;
        const int x0 = xseg * TM;

        float d[NB][R];
#pragma unroll 1
        for (int c = 0; c < NC; ++c, ++g) {
            const int b = (int)(g & 1u);
            if (g >= 2) {
                // this warpgroup's MMAs of chunk g-2 have finished reading A[b] and their weight slot; the CTA barrier makes
                // that true of both warpgroups (chunk g-1 may still run)
                if (c > 0) wg_wait<1>();
                __syncthreads();
                if (warp == 0) {
                    if (g + 2 < g_total && elect_one()) {   // refill that slot with chunk g+2
                        const uint32_t q = g + 2, slot = q % RING;
                        mbar_expect_tx(&s.bar_wfull[slot], WCHUNK);
                        bulk_g2s(s.w[slot], a.wt + (size_t)(q % NC) * WCHUNK, WCHUNK, &s.bar_wfull[slot]);
                    }
                    __syncwarp();
                }
            }
            // ---- A[b] <- the 128 x 64 window of tap (dy, dx), channel block cb ----
            {
                const int tap = c / CB, cb = c - tap * CB;
                const int dy = tap / 3 - 1, dx = tap - (tap / 3) * 3 - 1;
                const int yy = y + dy;
                const bool row_ok = (unsigned)yy < (unsigned)a.H;
                const __half *src = a.in + ((size_t)(f * a.H + (row_ok ? yy : 0)) * a.W) * CIN + cb * 64;
                uint4 v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int q = j * NT + tid, row = q >> 3, ch = q & 7, xx = x0 + row + dx;
                    v[j] = make_uint4(0u, 0u, 0u, 0u);
                    if (row_ok && (unsigned)xx < (unsigned)a.W) v[j] = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)xx * CIN) + ch);
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int q = j * NT + tid, row = q >> 3, ch = q & 7;
                    *reinterpret_cast<uint4 *>(s.a[b] + sw128_off(row, ch)) = v[j];
                }
            }
            fence_async_smem();
            __syncthreads();
            {
                const uint32_t slot = g % RING;
                mbar_wait(&s.bar_wfull[slot], (g / RING) & 1u);
                const uint32_t a_addr = smem_u32(s.a[b]) + (uint32_t)wg * SW128_HALF, w_addr = smem_u32(s.w[slot]);
                wg_fence();
#pragma unroll
                for (int nb = 0; nb < NB; ++nb)
                    wgmma_sw<NROWS, false>(d[nb], a_addr, w_addr + (uint32_t)(nb * NROWS * 128), 4, c > 0 ? 1u : 0u);
                wg_commit();
            }
        }
        wg_wait<0>();
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) acc_fence(d[nb]);

        // ================= epilogue of the tile (accumulator fragment: rows 64*wg + frag_row, columns frag_col) =================
        if (LAYER == 0 || LAYER == 2) {
            float dot[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
            float nz[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int x = x0 + 64 * wg + frag_row(2 * h, lane, wwarp);
                nz[h] = a.noise ? __ldg(a.noise + (size_t)f * a.noise_fstride + (size_t)y * a.W + x) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < R; i += 2) {
                const int h = (i >> 1) & 1, col = frag_col(i, lane);
                const float t0 = lrelu_clamp(d[0][i] + nz[h] + s.bias[col]), t1 = lrelu_clamp(d[0][i + 1] + nz[h] + s.bias[col + 1]);
#pragma unroll
                for (int o = 0; o < 3; ++o) dot[h][o] = fmaf(t1, s.rgbw[o * COUT + col + 1], fmaf(t0, s.rgbw[o * COUT + col], dot[h][o]));
                if (LAYER == 0 || a.out) {   // LAYER 2 keeps its activation only for the backward (gfpp_sr_forward_train)
                    const size_t pix = ((size_t)f * a.H + y) * a.W + x0 + 64 * wg + frag_row(i, lane, wwarp);
                    *reinterpret_cast<uint32_t *>(a.out + pix * COUT + col) = pack2<false>(t0, t1);
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int o = 0; o < 3; ++o) {
                    float v = dot[h][o];
                    v += __shfl_xor_sync(0xffffffffu, v, 1);
                    v += __shfl_xor_sync(0xffffffffu, v, 2);
                    if ((lane & 3) == 0) s.part[o * TM + 64 * wg + frag_row(2 * h, lane, wwarp)] = v;
                }
            }
            __syncthreads();
            if (tid < TM) {
                const int x = x0 + tid;
                if (LAYER == 0) {   // toRGB (+ bias, clamp) added to the rgb skip (networks_stylegan2.py:395-403, 462-466)
                    const size_t pix = ((size_t)f * a.H + y) * a.W + x;
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        float r = s.part[o * TM + tid] + __ldg(a.rgb_b + o);
                        r = fminf(fmaxf(r, -256.f), 256.f);
                        a.img_out[pix * 3 + o] = __ldg(a.img_in + pix * 3 + o) + r;
                    }
                } else {
                    float sk[3], rc[3];
                    upsampled_skip(a.img_in + (size_t)f * (a.H / 2) * (a.W / 2) * 3, a.H / 2, a.W / 2, y, x, sk);
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        float r = s.part[o * TM + tid] + __ldg(a.rgb_b + o);
                        r = sk[o] + fminf(fmaxf(r, -256.f), 256.f);
                        rc[o] = fminf(fmaxf(r, 0.f), 1.f);
                        if (a.img_out) a.img_out[(((size_t)f * 3 + o) * a.H + y) * a.W + x] = a.clamp01 ? rc[o] : r;
                    }
                    if (a.img_u8) {
                        // video frame (rgb * 255).int() of the clamped colour, the rule of k_epilogue and dist.to_uint8.  A pixel is 3
                        // bytes: the tile's 128 pixels are staged in `part` (once this warpgroup has read it) and leave as 96 words
                        wg_sync(1);
                        unsigned char *stage = reinterpret_cast<unsigned char *>(s.part);
#pragma unroll
                        for (int o = 0; o < 3; ++o) stage[3 * tid + o] = (unsigned char)(int)__fmul_rn(rc[o], 255.0f);
                        wg_sync(1);
                        if (tid < 3 * TM / 4) {
                            uint32_t *dst = reinterpret_cast<uint32_t *>(a.img_u8 + (((size_t)f * a.H + y) * a.W + x0) * 3);
                            dst[tid] = reinterpret_cast<const uint32_t *>(stage)[tid];
                        }
                    }
                }
            }
        } else {
            // N-block `nb` holds the phases (py = nb, px = column / 64): output pixels (2y + py, 2x + px), 64 channels each
            const int Ho = 2 * a.H, Wo = 2 * a.W;
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
                for (int i = 0; i < R; i += 2) {
                    const int col = frag_col(i, lane), px = col >> 6, ch = col & 63;
                    const int x = x0 + 64 * wg + frag_row(i, lane, wwarp), Y = 2 * y + nb, X = 2 * x + px;
                    const size_t opix = ((size_t)f * Ho + Y) * Wo + X;
                    const float nz = a.noise ? __ldg(a.noise + (size_t)f * a.noise_fstride + (size_t)Y * Wo + X) : 0.f;
                    const float t0 = lrelu_clamp(d[nb][i] + nz + s.bias[ch]), t1 = lrelu_clamp(d[nb][i + 1] + nz + s.bias[ch + 1]);
                    *reinterpret_cast<uint32_t *>(a.out + opix * COUT + ch) = pack2<false>(t0, t1);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// block0.conv0: 3 -> 128 channels.  One task = two horizontally adjacent pixels x 16 output channels.  A warp takes ONE group of 16
// channels for 32 neighbouring pixel pairs, so every shared-memory weight read is a broadcast (one 16-byte wavefront instead of eight:
// spreading the eight channel groups over the lanes instead makes those reads the bound); the eight warps of a CTA cover the eight channel groups of the same 64 pixels.
__global__ void __launch_bounds__(256) k_sr_conv_in(const __grid_constant__ SrConvInArgs a) {
    __shared__ __align__(16) float sw[27 * 128];
    __shared__ float sb[128];
    for (int i = threadIdx.x; i < 27 * 128; i += 256) sw[i] = a.w[i];
    if (threadIdx.x < 128) sb[threadIdx.x] = a.bias[threadIdx.x];
    __syncthreads();
    const int Wh = a.W / 2;
    const long long n_groups = (long long)a.F * a.H * Wh / 32;       // groups of 32 pixel pairs (W % 64 == 0)
    const int cg = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (long long grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
        const long long pp = grp * 32 + lane;
        const int xh = (int)(pp % Wh);
        const long long r = pp / Wh;
        const int y = (int)(r % a.H), f = (int)(r / a.H);
        const int x = 2 * xh;
        float in[3][4][3];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int yy = y + ky - 1;
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) {
                const int xx = x + kx - 1;
                const bool ok = (unsigned)yy < (unsigned)a.H && (unsigned)xx < (unsigned)a.W;
                const float *p = a.in + (((size_t)f * a.H + (ok ? yy : 0)) * a.W + (ok ? xx : 0)) * 3;
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) in[ky][kx][ci] = ok ? __ldg(p + ci) : 0.f;
            }
        }
        float acc[2][16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[0][i] = acc[1][i] = 0.f;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const int k = (ky * 3 + kx) * 3 + ci;
                    const float4 *wp = reinterpret_cast<const float4 *>(sw + k * 128 + cg * 16);
                    const float a0 = in[ky][kx][ci], a1 = in[ky][kx + 1][ci];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float4 w4 = wp[q];
                        acc[0][4 * q + 0] = fmaf(a0, w4.x, acc[0][4 * q + 0]); acc[1][4 * q + 0] = fmaf(a1, w4.x, acc[1][4 * q + 0]);
                        acc[0][4 * q + 1] = fmaf(a0, w4.y, acc[0][4 * q + 1]); acc[1][4 * q + 1] = fmaf(a1, w4.y, acc[1][4 * q + 1]);
                        acc[0][4 * q + 2] = fmaf(a0, w4.z, acc[0][4 * q + 2]); acc[1][4 * q + 2] = fmaf(a1, w4.z, acc[1][4 * q + 2]);
                        acc[0][4 * q + 3] = fmaf(a0, w4.w, acc[0][4 * q + 3]); acc[1][4 * q + 3] = fmaf(a1, w4.w, acc[1][4 * q + 3]);
                    }
                }
            }
        }
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const size_t pix = ((size_t)f * a.H + y) * a.W + x + p;
            const float nz = a.noise ? __ldg(a.noise + (size_t)f * a.noise_fstride + (size_t)y * a.W + x + p) : 0.f;
            uint4 u[2];
            uint32_t *uw = reinterpret_cast<uint32_t *>(u);
#pragma unroll
            for (int i = 0; i < 8; ++i)
                uw[i] = pack2<false>(lrelu_clamp(acc[p][2 * i] + nz + sb[cg * 16 + 2 * i]), lrelu_clamp(acc[p][2 * i + 1] + nz + sb[cg * 16 + 2 * i + 1]));
            uint4 *dst = reinterpret_cast<uint4 *>(a.out + pix * 128 + cg * 16);
            dst[0] = u[0];
            dst[1] = u[1];
        }
    }
}

cudaError_t launch_sr_conv_in(const SrConvInArgs &a, cudaStream_t st) {
    if (a.W % 64) return cudaErrorInvalidValue;
    const uint64_t n_tasks = (uint64_t)a.F * a.H * (a.W / 2) * 8;   // one CTA iteration = 32 pixel pairs x 8 channel groups
    k_sr_conv_in<<<grid_for(n_tasks, 256), 256, 0, st>>>(a);
    return cudaGetLastError();
}

template <int LAYER>
static cudaError_t launch_sr_conv_t(const SrConvArgs &a, cudaStream_t st) {
    static_assert(sizeof(SmemSR<LAYER>) + 1024 <= 227 * 1024, "SR conv kernel exceeds the per-CTA shared memory limit");
    const size_t smem = sizeof(SmemSR<LAYER>) + 1024;
    // function attributes are per device: set on every launch, never cached process-wide
    cudaError_t e = cudaFuncSetAttribute(k_sr_conv<LAYER>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(k_sr_conv<LAYER>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    const int n_tiles = a.F * a.H * (a.W / TM);
    int per_sm = (int)((227 * 1024) / smem);                        // by shared memory
    if (per_sm > (LAYER == 1 ? 1 : 2)) per_sm = LAYER == 1 ? 1 : 2;  // the launch bound (registers)
    if (per_sm < 1) per_sm = 1;
    int blocks = sm_count() * per_sm;
    if (blocks > n_tiles) blocks = n_tiles;
    if (blocks < 1) return cudaErrorInvalidValue;
    k_sr_conv<LAYER><<<blocks, NT, smem, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sr_conv(int layer, const SrConvArgs &a, cudaStream_t st) {
    if (a.W % TM || a.F <= 0 || a.H <= 0) return cudaErrorInvalidValue;
    if (layer == 0) return launch_sr_conv_t<0>(a, st);
    if (layer == 1) return launch_sr_conv_t<1>(a, st);
    if (layer == 2) return launch_sr_conv_t<2>(a, st);
    return cudaErrorInvalidValue;
}

}  // namespace gfpp
