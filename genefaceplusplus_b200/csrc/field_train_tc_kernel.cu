// field_train_tc_kernel.cu -- RADNeRF.forward (modules/radnerfs/radnerf.py:108-141) and its backward for the training step on
// tensor cores: fp16 wgmma operands, fp32 accumulation, fp32 parameters in, fp32 gradients out.  The fp32 FFMA field
// (field_train_kernel.cu) computes the same function and is the reference this one is tested against.
//
// Shape of the computation
//   * a tile is 128 points; 256 threads = two warpgroups, warpgroup g owns points 64g..64g+63 of every [points x features] product;
//   * activations live in shared memory as fp16 SW128 tiles of [128 points x 64 features] (tc.cuh); the six wide layers' weights
//     are fp16 images of the same tile format that k_field_tc_relayout writes once per call (the weights change every step) and
//     every GEMM copies into shared memory;
//   * rounding sites: the operands of the wide products only -- grid features, SH, hidden activations, weights, and in the backward
//     the output gradients dY.  Accumulators, biases, ReLU / tanh / exp / sigmoid and their derivatives, the grid gathers and
//     scatters and the three narrow layers (ambient logits, the sigma row h0, colour logits) are fp32; the narrow layers read the
//     fp32 accumulators of the layer below, so the inputs of tanh and exp are never rounded to 16 bits;
//   * every dY block is multiplied by a power of two chosen from its largest magnitude before it is rounded to fp16 and the fp32
//     accumulator of each product with it is multiplied by the inverse, so the gradients are the same numbers times 2^k when the
//     upstream gradients are scaled by 2^k (loss scaling), and tiny upstream gradients are not flushed;
//   * input gradients dX = dY W: A = dY tile (K = outputs), B = the transposed weight image;
//     weight gradients dW = dY^T X: both operands are point-major tiles, read through MN-major descriptors (tc::desc_sw128_mn) with
//     K = the tile's 128 points; warpgroup g computes output rows 64g..64g+63;
//   * the determinism scheme of k_field_bwd: each persistent CTA owns a contiguous tile range and a FieldPart block of partial sums
//     (every element has one owner thread); k_field_reduce sums the blocks in CTA order.  The backward recomputes its tile's forward.
#include "common.cuh"
#include "field_train_tc_kernel.cuh"
#include "grid_train.cuh"
#include "launch.cuh"
#include "tc.cuh"

namespace gfpp {

namespace {

using namespace tc;

constexpr int TP = FIELD_TC_TP;
constexpr int NT = 256;
constexpr uint32_t T = FieldTcImg::T;

struct Smem {
    unsigned char X0[3 * T];      // colour net input: [geo 0:64 | geo 64:128 | SH 16, rest 0]; later the geo gradient
    unsigned char B1[2 * T];
    unsigned char B2[2 * T];
    unsigned char PA[T];          // [position features 32 | ambient features 32]
    unsigned char W[3 * T];       // the current product's weight image
    float stash[16 * NT];         // position-feature gradient of the sigma net, kept per thread until the ambient net adds its part
    float pt[TP * 4];
    float dr[TP * 4];
    float amb[TP * 4];            // tanh outputs
    float g3[TP * 4];             // colours, then colour / ambient logit gradients
    float h0[TP];
    float gh0[TP];
    float red[8];
    int valid[TP];
};

__device__ __forceinline__ uint32_t tile_off(int row, int col) { return (uint32_t)(col >> 6) * T + sw128_off(row, (col & 63) >> 3) + (uint32_t)(col & 7) * 2u; }
__device__ __forceinline__ void st2(unsigned char *tile, int row, int col, float a, float b) {
    *reinterpret_cast<uint32_t *>(tile + tile_off(row, col)) = pack2<false>(a, b);
}
__device__ __forceinline__ float2 ld2(const unsigned char *tile, int row, int col) {
    return __half22float2(*reinterpret_cast<const __half2 *>(tile + tile_off(row, col)));
}
__device__ __forceinline__ float ld1(const unsigned char *tile, int row, int col) {
    return __half2float(*reinterpret_cast<const __half *>(tile + tile_off(row, col)));
}

// Copies a weight image into s.W.  The leading barrier ends every read of s.W and of the activation tiles by the product before;
// the trailing fence + barrier publish the copy and every tile store since then to the tensor cores.
__device__ __forceinline__ void load_w(Smem &s, const unsigned char *__restrict__ img, uint32_t bytes, int tid) {
    __syncthreads();
    for (uint32_t i = (uint32_t)tid * 16u; i < bytes; i += NT * 16u) *reinterpret_cast<uint4 *>(s.W + i) = __ldg(reinterpret_cast<const uint4 *>(img + i));
    fence_async_smem();
    __syncthreads();
}

// D[64 x N] = A[64 x 16 KS] W^T: A = this warpgroup's half of consecutive activation tiles, W = s.W with K-tiles `wstride` apart
template <int N, int KS>
__device__ __forceinline__ void mma_k(float (&d)[N / 2], uint32_t a, uint32_t w, uint32_t wstride) {
    acc_zero(d);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
        wgmma<N, false>(d, desc_sw128(a + (uint32_t)(ks >> 2) * T + (uint32_t)(ks & 3) * 32u), desc_sw128(w + (uint32_t)(ks >> 2) * wstride + (uint32_t)(ks & 3) * 32u),
                        ks > 0 ? 1u : 0u);
    wg_commit();
    wg_wait<0>();
    acc_fence(d);
}

// D[64 x N] = Y^T X over the tile's 128 points: Y = one [128 x 64] tile (this warpgroup's 64 output rows), X = N / 64 consecutive tiles
template <int N>
__device__ __forceinline__ void mma_t(float (&d)[N / 2], uint32_t y, uint32_t x) {
    acc_zero(d);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < TP / 16; ++ks) wgmma_tn<N>(d, desc_sw128_mn(y + (uint32_t)ks * 2048u, T), desc_sw128_mn(x + (uint32_t)ks * 2048u, T), ks > 0 ? 1u : 0u);
    wg_commit();
    wg_wait<0>();
    acc_fence(d);
}

// part[n][col0 + c] += inv * D[n][c] for c < ncols; n = this warpgroup's rows.  Each element has one owner thread.
template <int N>
__device__ __forceinline__ void add_part(const float (&d)[N / 2], float inv, float *__restrict__ part, int ldp, int ncols, int tid) {
    const int lane = tid & 31, wwarp = (tid >> 5) & 3, wg = tid >> 7;
#pragma unroll
    for (int i = 0; i < N / 2; i += 2) {
        const int n = 64 * wg + frag_row(i, lane, wwarp), c = frag_col(i, lane);
        if (c < ncols) {
            float2 *q = reinterpret_cast<float2 *>(part + (size_t)n * ldp + c);
            float2 v = *q;
            v.x = fmaf(d[i], inv, v.x);
            v.y = fmaf(d[i + 1], inv, v.y);
            *q = v;
        }
    }
}

// The CTA's power of two 2^k that brings `mx` (this thread's largest magnitude) of the whole block to [256, 512), and its inverse;
// 1 when the block is all zero or not finite.
__device__ __forceinline__ float block_scale(Smem &s, float mx, int tid, float &inv) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) s.red[tid >> 5] = mx;
    __syncthreads();
    float m = s.red[0];
#pragma unroll
    for (int i = 1; i < NT / 32; ++i) m = fmaxf(m, s.red[i]);
    __syncthreads();
    int k = 0;
    if (m > 0.f && m < INFINITY) k = min(126, max(-126, 135 - ((__float_as_int(m) >> 23) & 255)));
    inv = __int_as_float((127 - k) << 23);
    return __int_as_float((127 + k) << 23);
}

// Rounds a [128 x 128] block of gradients held in accumulator fragments to fp16 under the block's scale; returns the inverse scale.
__device__ __forceinline__ float scale_store(Smem &s, const float (&d)[64], unsigned char *out, int tid) {
    const int lane = tid & 31, wwarp = (tid >> 5) & 3, wg = tid >> 7;
    float mx = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) mx = fmaxf(mx, fabsf(d[i]));
    float inv;
    const float sc = block_scale(s, mx, tid, inv);
#pragma unroll
    for (int i = 0; i < 64; i += 2) st2(out, 64 * wg + frag_row(i, lane, wwarp), frag_col(i, lane), d[i] * sc, d[i + 1] * sc);
    return inv;
}

// ReLU (optional) of an accumulator block, stored as an fp16 activation tile pair
__device__ __forceinline__ void act_store(float (&d)[64], const float *__restrict__ bias, bool relu, unsigned char *out, int tid) {
    const int lane = tid & 31, wwarp = (tid >> 5) & 3, wg = tid >> 7;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int c = frag_col(i, lane);
        if (bias) { d[i] += bias[c]; d[i + 1] += bias[c + 1]; }
        if (relu) { d[i] = fmaxf(d[i], 0.f); d[i + 1] = fmaxf(d[i + 1], 0.f); }
        st2(out, 64 * wg + frag_row(i, lane, wwarp), c, d[i], d[i + 1]);
    }
}

// Narrow layer on the fp32 accumulators: o[r][j] = sum_k D[row r][k] W[j][k] for the thread's two rows (frag_row(0), frag_row(2)),
// complete in all four lanes that share the rows; fixed order.
template <int NO>
__device__ __forceinline__ void narrow_acc(const float (&d)[64], const float *__restrict__ W, int no, int lane, float (&o)[2][NO]) {
#pragma unroll
    for (int j = 0; j < NO; ++j) {
        float v0 = 0.f, v1 = 0.f;
        if (j < no) {
#pragma unroll
            for (int i = 0; i < 64; i += 4) {
                const float2 w = __ldg(reinterpret_cast<const float2 *>(W + j * 128 + frag_col(i, lane)));
                v0 = fmaf(d[i], w.x, v0);
                v0 = fmaf(d[i + 1], w.y, v0);
                v1 = fmaf(d[i + 2], w.x, v1);
                v1 = fmaf(d[i + 3], w.y, v1);
            }
        }
        v0 += __shfl_xor_sync(0xffffffffu, v0, 1);
        v0 += __shfl_xor_sync(0xffffffffu, v0, 2);
        v1 += __shfl_xor_sync(0xffffffffu, v1, 1);
        v1 += __shfl_xor_sync(0xffffffffu, v1, 2);
        o[0][j] = v0;
        o[1][j] = v1;
    }
}

// Narrow layer weight gradient: part[o][k] += sum_p g[p * gs + o] * X[p][k], o < no, k < 128; X an activation tile pair.
__device__ __forceinline__ void narrow_dw(const float *g, int gs, const unsigned char *X, int no, float *__restrict__ part, int tid) {
    for (int e = tid; e < no * 128; e += NT) {
        const int o = e >> 7, k = e & 127;
        float v = 0.f;
        for (int p = 0; p < TP; ++p) v = fmaf(g[p * gs + o], ld1(X, p, k), v);
        part[e] += v;
    }
}

// Narrow layer input gradient through the ReLU of activation tile pair X, in place: X[p][k] <- fp16(scale * (X[p][k] > 0 ? sum_o
// g[p][o] W[o][k] : 0)); returns the inverse scale.
__device__ __forceinline__ float narrow_dx_relu(Smem &s, const float *g, unsigned char *X, const float *__restrict__ W, int no, int tid) {
    auto val = [&](int e) {
        const int p = e >> 6, k = (e & 63) * 2;
        const float2 x = ld2(X, p, k);
        float2 v = make_float2(0.f, 0.f);
        for (int o = 0; o < no; ++o) {
            const float2 w = __ldg(reinterpret_cast<const float2 *>(W + o * 128 + k));
            v.x = fmaf(g[p * 4 + o], w.x, v.x);
            v.y = fmaf(g[p * 4 + o], w.y, v.y);
        }
        if (!(x.x > 0.f)) v.x = 0.f;
        if (!(x.y > 0.f)) v.y = 0.f;
        return v;
    };
    float mx = 0.f;
    for (int e = tid; e < TP * 64; e += NT) {
        const float2 v = val(e);
        mx = fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y)));
    }
    float inv;
    const float sc = block_scale(s, mx, tid, inv);
    for (int e = tid; e < TP * 64; e += NT) {
        const float2 v = val(e);
        st2(X, e >> 6, (e & 63) * 2, v.x * sc, v.y * sc);
    }
    return inv;
}

// column sums over the tile: part[n] += inv * sum_p Y[p][n]
__device__ __forceinline__ void colsum(const unsigned char *Y, float inv, float *__restrict__ part, int tid) {
    if (tid < 128) {
        float v = 0.f;
        for (int p = 0; p < TP; ++p) v += ld1(Y, p, tid);
        part[tid] = fmaf(v, inv, part[tid]);
    }
}

__device__ __forceinline__ void to_unit(const float *x, float bound, float *u) {
    const float twob = 2.0f * bound;
    for (int d = 0; d < 3; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], bound), twob);
}

// the ambient net up to its second hidden layer: PA[:, 0:32] -> B1 = hidden 1 -> accumulators d = hidden 2 (after the ReLU)
__device__ __forceinline__ void ambient_hidden(const FieldTcArgs &A, Smem &s, float (&d)[64], int tid) {
    const uint32_t half = (uint32_t)(tid >> 7) * SW128_HALF;
    load_w(s, A.img + FieldTcImg::a0, T, tid);
    mma_k<128, 2>(d, smem_u32(s.PA) + half, smem_u32(s.W), T);
    act_store(d, A.f.wt, true, s.B1, tid);
    load_w(s, A.img + FieldTcImg::a1, 2 * T, tid);
    mma_k<128, 8>(d, smem_u32(s.B1) + half, smem_u32(s.W), T);
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = fmaxf(d[i], 0.f);
}

// ---- the forward of one tile; leaves X0 = [geo | SH], B1 = colour hidden, B2 = sigma hidden 2, PA = [pos | ambient] features,
//      amb / h0 / g3 = tanh outputs, the sigma row, colours ----
__device__ void tile_forward(const FieldTcArgs &A, Smem &s, uint32_t tile, int tid, bool write_out) {
    const FieldArgs &a = A.f;
    const uint32_t base = tile * TP;
    const int lane = tid & 31, wwarp = (tid >> 5) & 3, wg = tid >> 7;
    const uint32_t half = (uint32_t)wg * SW128_HALF;
    const int r0 = 64 * wg + frag_row(0, lane, wwarp), r1 = r0 + 8;
    if (tid < TP) {
        const uint32_t p = base + tid;
        const bool v = p < a.M;
        s.valid[tid] = v;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            s.pt[tid * 4 + d] = v ? a.xyzs[(size_t)p * 3 + d] : 0.f;
            s.dr[tid * 4 + d] = v ? a.dirs[(size_t)p * 3 + d] : 0.f;
        }
    }
    __syncthreads();
    const int p = tid & (TP - 1), lg = tid >> 7;
    // position grid -> PA[:, 0:32]
    {
        float u[3];
        to_unit(s.pt + p * 4, a.bound, u);
        for (int l = lg * 8; l < lg * 8 + 8; ++l) {
            const float2 f = s.valid[p] ? grid_lookup3(a.pos_gm, a.pos_tab, l, u[0], u[1], u[2]) : make_float2(0.f, 0.f);
            st2(s.PA, p, 2 * l, f.x, f.y);
        }
    }
    float d[64];
    // ambient net (conditioning folded into the first layer's bias) -> tanh of the fp32 logits
    ambient_hidden(A, s, d, tid);
    {
        float o[2][3];
        narrow_acc<3>(d, a.w[2], a.amb_dim, lane, o);
        if ((lane & 3) == 0)
            for (int j = 0; j < a.amb_dim; ++j) {
                s.amb[r0 * 4 + j] = tanhf(o[0][j]);
                s.amb[r1 * 4 + j] = tanhf(o[1][j]);
            }
    }
    __syncthreads();
    // ambient grid (bound 1) -> PA[:, 32:64]
    {
        float u[3] = {0.f, 0.f, 0.f};
        for (int j = 0; j < a.amb_dim; ++j) u[j] = __fdiv_rn(__fadd_rn(s.amb[p * 4 + j], 1.0f), 2.0f);
        for (int l = lg * 8; l < lg * 8 + 8; ++l) {
            float2 f = make_float2(0.f, 0.f);
            if (s.valid[p]) f = a.amb_dim == 3 ? grid_lookup3(a.amb_gm, a.amb_tab, l, u[0], u[1], u[2]) : grid_lookup2(a.amb_gm, a.amb_tab, l, u[0], u[1]);
            st2(s.PA, p, 32 + 2 * l, f.x, f.y);
        }
    }
    // sigma net; the sigma row h0 from the fp32 accumulators
    load_w(s, A.img + FieldTcImg::s0, T, tid);
    mma_k<128, 4>(d, smem_u32(s.PA) + half, smem_u32(s.W), T);
    act_store(d, nullptr, true, s.B1, tid);
    load_w(s, A.img + FieldTcImg::s1, 2 * T, tid);
    mma_k<128, 8>(d, smem_u32(s.B1) + half, smem_u32(s.W), T);
    act_store(d, nullptr, true, s.B2, tid);
    {
        float o[2][1];
        narrow_acc<1>(d, a.w[5], 1, lane, o);
        if ((lane & 3) == 0) {
            s.h0[r0] = o[0][0];
            s.h0[r1] = o[1][0];
        }
    }
    load_w(s, A.img + FieldTcImg::s2, 2 * T, tid);
    mma_k<128, 8>(d, smem_u32(s.B2) + half, smem_u32(s.W), T);
    act_store(d, nullptr, false, s.X0, tid);   // geo features
    if (tid < TP) {   // SH(dir) -> X0 tile 2, columns 0..15
        float sh[16];
        sh4(s.dr[tid * 4], s.dr[tid * 4 + 1], s.dr[tid * 4 + 2], sh);
        for (int j = 0; j < 16; j += 2) st2(s.X0, tid, 128 + j, sh[j], sh[j + 1]);
    }
    // colour net (individual code folded into the first layer's bias) -> sigmoid of the fp32 logits
    load_w(s, A.img + FieldTcImg::c0, 3 * T, tid);
    mma_k<128, 9>(d, smem_u32(s.X0) + half, smem_u32(s.W), T);
    act_store(d, a.wt + 128, true, s.B1, tid);
    {
        float o[2][3];
        narrow_acc<3>(d, a.w[7], 3, lane, o);
        if ((lane & 3) == 0)
            for (int c = 0; c < 3; ++c) {
                s.g3[r0 * 4 + c] = 1.0f / (1.0f + expf(-o[0][c]));
                s.g3[r1 * 4 + c] = 1.0f / (1.0f + expf(-o[1][c]));
            }
    }
    __syncthreads();
    if (write_out && tid < TP && s.valid[tid]) {
        const size_t q = base + tid;
        a.sigma[q] = expf(s.h0[tid]);   // trunc_exp forward is plain exp (utils.py:36-41); density_scale is the caller's
        for (int c = 0; c < 3; ++c) a.color[q * 3 + c] = s.g3[tid * 4 + c];
        for (int j = 0; j < a.amb_dim; ++j) a.ambient[q * a.amb_dim + j] = s.amb[tid * 4 + j];
    }
    __syncthreads();
}

__device__ __forceinline__ Smem &smem_struct(unsigned char *raw) {
    return *reinterpret_cast<Smem *>(raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u));   // SW128 tiles need 1024-byte alignment
}

// columns 16..63 of X0's SH tile are never written by a tile's forward: zero them once (they are operands of the colour net's weight
// gradient, whose columns past 16 are dropped)
__device__ __forceinline__ void zero_sh_tile(Smem &s, int tid) {
    for (uint32_t i = (uint32_t)tid * 16u; i < T; i += NT * 16u) *reinterpret_cast<uint4 *>(s.X0 + 2 * T + i) = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
}

}  // namespace

// fp16 weight images (FieldTcImg) and the two folded fp32 biases; blockIdx.y selects the image, one thread per element
__global__ void k_field_tc_relayout(const __grid_constant__ FieldTcArgs A) {
    const FieldArgs &a = A.f;
    const int ldc0 = 144 + a.ind_dim;
    // image (rows x 64 * kt): element (r, k) = W[r0 + r][c0 + k] (r < nr, k < nc), or transposed W[r0 + k][c0 + r] (k < nr, r < nc)
    struct Img { uint32_t off; int w, ld, r0, c0, nr, nc, tr, rows, kt; };
    const Img imgs[13] = {
        {FieldTcImg::a0, 0, 96, 0, 0, 128, 32, 0, 128, 1},        {FieldTcImg::a1, 1, 128, 0, 0, 128, 128, 0, 128, 2},
        {FieldTcImg::s0, 3, 64, 0, 0, 128, 64, 0, 128, 1},        {FieldTcImg::s1, 4, 128, 0, 0, 128, 128, 0, 128, 2},
        {FieldTcImg::s2, 5, 128, 1, 0, 128, 128, 0, 128, 2},      {FieldTcImg::c0, 6, ldc0, 0, 16, 128, 128, 0, 128, 2},
        {FieldTcImg::c0 + 2 * T, 6, ldc0, 0, 0, 128, 16, 0, 128, 1}, {FieldTcImg::c0T, 6, ldc0, 0, 16, 128, 128, 1, 128, 2},
        {FieldTcImg::s2T, 5, 128, 1, 0, 128, 128, 1, 128, 2},     {FieldTcImg::s1T, 4, 128, 0, 0, 128, 128, 1, 128, 2},
        {FieldTcImg::s0T, 3, 64, 0, 0, 128, 64, 1, 64, 2},        {FieldTcImg::a1T, 1, 128, 0, 0, 128, 128, 1, 128, 2},
        {FieldTcImg::a0T, 0, 96, 0, 0, 128, 32, 1, 64, 2}};
    const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    if (blockIdx.y == 13) {
        float *bias = reinterpret_cast<float *>(A.img + FieldTcImg::bias);
        for (uint32_t i = t0; i < 256; i += stride) {
            const uint32_t n = i & 127;
            float v = 0.f;
            if (i < 128) for (int k = 0; k < 64; ++k) v = fmaf(a.cond[k], a.w[0][n * 96 + 32 + k], v);
            else for (int j = 0; j < a.ind_dim; ++j) v = fmaf(a.code[j], a.w[6][n * ldc0 + 144 + j], v);
            bias[i] = v;
        }
        return;
    }
    const Img im = imgs[blockIdx.y];
    const float *W = a.w[im.w];
    const uint32_t total = (uint32_t)im.rows * 64u * (uint32_t)im.kt;
    for (uint32_t i = t0; i < total; i += stride) {
        const int k = (int)(i % (64u * im.kt)), r = (int)(i / (64u * im.kt));
        float v = 0.f;
        if (!im.tr) { if (r < im.nr && k < im.nc) v = W[(size_t)(im.r0 + r) * im.ld + im.c0 + k]; }
        else if (k < im.nr && r < im.nc) v = W[(size_t)(im.r0 + k) * im.ld + im.c0 + r];
        const uint32_t off = im.off + (uint32_t)(k >> 6) * (uint32_t)im.rows * 128u + sw128_off(r, (k & 63) >> 3) + (uint32_t)(k & 7) * 2u;
        *reinterpret_cast<__half *>(A.img + off) = __float2half_rn(v);
    }
}

__global__ void __launch_bounds__(NT, 1) k_field_tc_fwd(const __grid_constant__ FieldTcArgs A) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Smem &s = smem_struct(smem_raw);
    const uint32_t n_tiles = (A.f.M + TP - 1) / TP;
    zero_sh_tile(s, threadIdx.x);
    for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) tile_forward(A, s, t, threadIdx.x, true);
}

// Backward of one tile after its forward (X0 = [geo | SH], B1 = c1, B2 = s2, PA = [pos | amb features]); g_x is the gradient of the
// pre-activation of x, stored fp16 under its block scale:
//   1 colour logits' gradient, dW c1;  2 g_c1 in place (B1);  3 column sums, dW c0;  4 g_geo = g_c1 W_c0[:, 16:144] -> X0
//   5 dW s2;  6 g_s2 in place (B2);  7 s1 recomputed -> B1;  8 dW s1;  9 g_s1 in place (B1);  10 dW s0
//   11 g_[pos|amb feat] = g_s1 W_s0 in registers: position half -> stash;  12 ambient grid: table scatter, input gradient, tanh'
//   13 a1 -> B1, a2 -> B2 recomputed;  14 dW a2, g_a2 in place (B2);  15 dW a1;  16 g_a1 in place (B1), column sums, dW a0
//   17 g_pos = stash + g_a1 W_a0[:, 0:32];  18 position grid: table scatter
__global__ void __launch_bounds__(NT, 1) k_field_tc_bwd(const __grid_constant__ FieldTcArgs A) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Smem &s = smem_struct(smem_raw);
    const FieldArgs &a = A.f;
    const int tid = threadIdx.x, lane = tid & 31, wwarp = (tid >> 5) & 3, wg = tid >> 7, q4 = lane & 3;
    const uint32_t half = (uint32_t)wg * SW128_HALF;
    const int r0 = 64 * wg + frag_row(0, lane, wwarp);
    float *part = a.part + (size_t)blockIdx.x * FieldPart::total;
    for (size_t i = tid; i < FieldPart::total; i += NT) part[i] = 0.f;
    zero_sh_tile(s, tid);
    const uint32_t n_tiles = (a.M + TP - 1) / TP;
    const uint32_t t0 = (uint32_t)((uint64_t)n_tiles * blockIdx.x / gridDim.x), t1 = (uint32_t)((uint64_t)n_tiles * (blockIdx.x + 1) / gridDim.x);
    const uint32_t uX0 = smem_u32(s.X0), uB1 = smem_u32(s.B1), uB2 = smem_u32(s.B2), uPA = smem_u32(s.PA), uW = smem_u32(s.W);
    for (uint32_t t = t0; t < t1; ++t) {
        tile_forward(A, s, t, tid, false);
        const uint32_t base = t * TP;
        float d[64], e[32], inv;
        // 1: sigmoid' and trunc_exp' (exp of the clamped input, utils.py:43-47)
        if (tid < TP) {
            const bool v = s.valid[tid] != 0;
            for (int c = 0; c < 3; ++c) {
                const float y = s.g3[tid * 4 + c];
                const float g = v ? a.g_color[(size_t)(base + tid) * 3 + c] : 0.f;
                s.g3[tid * 4 + c] = g * (1.0f - y) * y;
            }
            s.gh0[tid] = v ? a.g_sigma[base + tid] * expf(clampf(s.h0[tid], -15.f, 15.f)) : 0.f;
        }
        __syncthreads();
        narrow_dw(s.g3, 4, s.B1, 3, part + FieldPart::c1, tid);
        __syncthreads();
        // 2
        inv = narrow_dx_relu(s, s.g3, s.B1, a.w[7], 3, tid);
        fence_async_smem();
        __syncthreads();
        // 3
        colsum(s.B1, inv, part + FieldPart::csc, tid);
        mma_t<128>(d, uB1 + (uint32_t)wg * T, uX0);
        add_part<128>(d, inv, part + FieldPart::c0 + 16, 144, 128, tid);
        mma_t<64>(e, uB1 + (uint32_t)wg * T, uX0 + 2 * T);
        add_part<64>(e, inv, part + FieldPart::c0, 144, 16, tid);
        // 4
        load_w(s, A.img + FieldTcImg::c0T, 2 * T, tid);
        mma_k<128, 8>(d, uB1 + half, uW, T);
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] *= inv;
        inv = scale_store(s, d, s.X0, tid);
        fence_async_smem();
        __syncthreads();
        // 5: the sigma row, then the geo rows
        narrow_dw(s.gh0, 1, s.B2, 1, part + FieldPart::s2, tid);
        mma_t<128>(d, uX0 + (uint32_t)wg * T, uB2);
        add_part<128>(d, inv, part + FieldPart::s2 + 128, 128, 128, tid);
        // 6: g_s2 = (g_geo W_s2[1:129] + g_h0 W_s2[0]) masked by s2 > 0
        load_w(s, A.img + FieldTcImg::s2T, 2 * T, tid);
        mma_k<128, 8>(d, uX0 + half, uW, T);
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int r = 64 * wg + frag_row(i, lane, wwarp), c = frag_col(i, lane);
            const float2 m = ld2(s.B2, r, c), w = __ldg(reinterpret_cast<const float2 *>(a.w[5] + c));
            d[i] = m.x > 0.f ? fmaf(s.gh0[r], w.x, d[i] * inv) : 0.f;
            d[i + 1] = m.y > 0.f ? fmaf(s.gh0[r], w.y, d[i + 1] * inv) : 0.f;
        }
        __syncthreads();   // every warpgroup has read its s2 rows
        inv = scale_store(s, d, s.B2, tid);
        // 7
        load_w(s, A.img + FieldTcImg::s0, T, tid);
        mma_k<128, 4>(d, uPA + half, uW, T);
        act_store(d, nullptr, true, s.B1, tid);
        fence_async_smem();
        __syncthreads();
        // 8
        mma_t<128>(d, uB2 + (uint32_t)wg * T, uB1);
        add_part<128>(d, inv, part + FieldPart::s1, 128, 128, tid);
        // 9
        load_w(s, A.img + FieldTcImg::s1T, 2 * T, tid);
        mma_k<128, 8>(d, uB2 + half, uW, T);
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const float2 m = ld2(s.B1, 64 * wg + frag_row(i, lane, wwarp), frag_col(i, lane));
            d[i] = m.x > 0.f ? d[i] * inv : 0.f;
            d[i + 1] = m.y > 0.f ? d[i + 1] * inv : 0.f;
        }
        __syncthreads();
        inv = scale_store(s, d, s.B1, tid);
        fence_async_smem();
        __syncthreads();
        // 10
        mma_t<64>(e, uB1 + (uint32_t)wg * T, uPA);
        add_part<64>(e, inv, part + FieldPart::s0, 64, 64, tid);
        // 11: accumulator column 8j + 2 q4 + f is feature f of level 4j + q4 (position grid, j < 4) or 4(j - 4) + q4 (ambient grid)
        load_w(s, A.img + FieldTcImg::s0T, T, tid);
        mma_k<64, 8>(e, uB1 + half, uW, T / 2);
#pragma unroll
        for (int i = 0; i < 16; ++i) s.stash[i * NT + tid] = e[i] * inv;
        // 12: ambient grid -- table gradient, input gradient through dy_dx, (x+1)/2 and tanh'
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            const int p = r0 + 8 * rs;
            float u[3] = {0.f, 0.f, 0.f};
            for (int j = 0; j < a.amb_dim; ++j) u[j] = __fdiv_rn(__fadd_rn(s.amb[p * 4 + j], 1.0f), 2.0f);
            float gin[3] = {0.f, 0.f, 0.f};
            if (s.valid[p]) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int l = 4 * j + q4;
                    const float2 g = make_float2(e[16 + 4 * j + 2 * rs] * inv, e[16 + 4 * j + 2 * rs + 1] * inv);
                    if (a.amb_dim == 3) {
                        grid_scatter<3>(a.amb_gm, l, u, g, a.g_amb_tab);
                        grid_input_grad<3>(a.amb_gm, a.amb_tab, l, u, g, gin);
                    } else {
                        grid_scatter<2>(a.amb_gm, l, u, g, a.g_amb_tab);
                        grid_input_grad<2>(a.amb_gm, a.amb_tab, l, u, g, gin);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                gin[j] += __shfl_xor_sync(0xffffffffu, gin[j], 1);
                gin[j] += __shfl_xor_sync(0xffffffffu, gin[j], 2);
            }
            if (q4 == 0)
                for (int j = 0; j < 3; ++j) {
                    float g = 0.f;
                    if (s.valid[p] && j < a.amb_dim) {
                        const float y = s.amb[p * 4 + j];
                        g = (gin[j] / 2.0f + a.g_ambient[(size_t)(base + p) * a.amb_dim + j]) * (1.0f - y * y);
                    }
                    s.g3[p * 4 + j] = g;
                }
        }
        // 13
        ambient_hidden(A, s, d, tid);
        act_store(d, nullptr, false, s.B2, tid);
        __syncthreads();
        // 14
        narrow_dw(s.g3, 4, s.B2, a.amb_dim, part + FieldPart::a2, tid);
        __syncthreads();
        inv = narrow_dx_relu(s, s.g3, s.B2, a.w[2], a.amb_dim, tid);
        fence_async_smem();
        __syncthreads();
        // 15
        mma_t<128>(d, uB2 + (uint32_t)wg * T, uB1);
        add_part<128>(d, inv, part + FieldPart::a1, 128, 128, tid);
        // 16
        load_w(s, A.img + FieldTcImg::a1T, 2 * T, tid);
        mma_k<128, 8>(d, uB2 + half, uW, T);
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const float2 m = ld2(s.B1, 64 * wg + frag_row(i, lane, wwarp), frag_col(i, lane));
            d[i] = m.x > 0.f ? d[i] * inv : 0.f;
            d[i + 1] = m.y > 0.f ? d[i + 1] * inv : 0.f;
        }
        __syncthreads();
        inv = scale_store(s, d, s.B1, tid);
        fence_async_smem();
        __syncthreads();
        colsum(s.B1, inv, part + FieldPart::csa, tid);
        mma_t<64>(e, uB1 + (uint32_t)wg * T, uPA);
        add_part<64>(e, inv, part + FieldPart::a0, 32, 32, tid);
        // 17
        load_w(s, A.img + FieldTcImg::a0T, T, tid);
        mma_k<64, 8>(e, uB1 + half, uW, T / 2);
        // 18: position grid -- table gradient only (xyzs never requires grad in the reference)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
            const int p = r0 + 8 * rs;
            if (s.valid[p]) {
                float u[3];
                to_unit(s.pt + p * 4, a.bound, u);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = 4 * j + 2 * rs;
                    grid_scatter<3>(a.pos_gm, 4 * j + q4, u, make_float2(fmaf(e[i], inv, s.stash[i * NT + tid]), fmaf(e[i + 1], inv, s.stash[(i + 1) * NT + tid])),
                                    a.g_pos_tab);
                }
            }
        }
        __syncthreads();
    }
}

cudaError_t launch_field_tc_relayout(const FieldTcArgs &a, cudaStream_t st) {
    k_field_tc_relayout<<<dim3(16, 14), 256, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_field_tc_fwd(const FieldTcArgs &a, cudaStream_t st) {
    const int smem = (int)sizeof(Smem) + 1024;
    cudaError_t e = cudaFuncSetAttribute(k_field_tc_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    const uint32_t n_tiles = (a.f.M + TP - 1) / TP;
    const int blocks = (int)(n_tiles < (uint32_t)sm_count() ? n_tiles : (uint32_t)sm_count());
    k_field_tc_fwd<<<blocks, NT, smem, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_field_tc_bwd(const FieldTcArgs &a, cudaStream_t st) {
    const int smem = (int)sizeof(Smem) + 1024;
    cudaError_t e = cudaFuncSetAttribute(k_field_tc_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    k_field_tc_bwd<<<a.f.n_cta, NT, smem, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gfpp
