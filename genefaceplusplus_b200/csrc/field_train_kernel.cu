// field_train_kernel.cu -- RADNeRF.forward (modules/radnerfs/radnerf.py:108-141) and its backward for the training step, fp32 FFMA.
//
//   position grid -> ambient net (96 -> 128 -> 128 -> A) -> tanh -> ambient grid -> sigma net (64 -> 128 -> 128 -> 129) -> exp
//   SH(dir) + geo features + individual code -> colour net (148 -> 128 -> 3) -> sigmoid
//
// Shape of the computation
//   * a tile is 64 points; 256 threads; every activation lives in shared memory in point-major rows;
//   * wide layers are 64x128xK FFMA tile GEMMs (gemm_pt): the A tile comes from shared memory, the weight operand is staged through
//     shared memory 32 k-rows at a time.  The forward reads the k-major transposes k_field_relayout writes into the workspace; the
//     backward's input gradients (dX = dY W) read the nn.Linear [out, in] weights in place, which are already k-major for that product;
//   * the conditioning vector and the individual code are the same for every point, so their columns of ambient_net.0 / color_net.0
//     are folded into bias vectors (forward), and their weight and input gradients follow from the column sums of the layer's output
//     gradient (k_field_reduce) -- no per-point copy of them is ever formed;
//   * the backward recomputes the forward of its tile (no per-point state is saved between the two calls), keeps three 64-row
//     activation buffers and the 64 grid features per point, and recomputes the ambient and the first sigma layer once more when their
//     buffers have been reused (see the step list in k_field_bwd);
//   * weight gradients: each persistent CTA owns a contiguous range of tiles and a block of partial sums in the workspace that its
//     threads update with plain read-modify-writes (each element has one owner thread); k_field_reduce sums the blocks in CTA order.
//     Nothing but the two table gradients depends on scheduling; those are scattered with float2 vector reductions, as the reference's
//     grid backward does.
#include "common.cuh"
#include "field_train_kernel.cuh"
#include "grid_train.cuh"
#include "launch.cuh"

namespace gfpp {

namespace {

constexpr int TP = FIELD_TP;
constexpr int NT = 256;
constexpr int LD0 = 148;      // B0 row stride: [SH 16 | geo 128] (+4 pad)
constexpr int LD1 = 132;      // B1 / B2 row stride
constexpr int LDPA = 68;      // PA row stride: [position features 32 | ambient features 32]
constexpr int KC = 32;        // weight k-rows staged per step

struct Smem {
    float B0[TP * LD0];
    float B1[TP * LD1];
    float B2[TP * LD1];
    float PA[TP * LDPA];
    float Wst[KC * 128];
    float pt[TP * 4];         // positions
    float dr[TP * 4];         // directions
    float amb[TP * 4];        // tanh outputs
    float g3[TP * 4];         // colour / ambient logit gradients
    float h0[TP];
    float gh0[TP];
    float gu[4 * TP * 4];     // ambient-grid input gradient, one partial per level group
    int valid[TP];
};

// Epilogue of a point-major tile GEMM: v = acc (+ bias[n]) (+ r1p[p] * r1w[n]); relu; masked by mask[p][n] > 0; (+= out); -> out[p][n]
struct Epi {
    const float *bias = nullptr;
    const float *r1p = nullptr, *r1w = nullptr;
    const float *mask = nullptr;
    int ldm = 0;
    bool relu = false, add = false;
};

// out[p][n] = epi(sum_k A[p][k] * B[k][n]) for p < 64, n < nout; A in shared memory (row stride lda), B global k-major with row stride
// ldb, columns >= width read as 0.  A, B, lda, ldb 16-byte aligned / multiples of 4; K a multiple of 4.
__device__ __forceinline__ void gemm_pt(Smem &s, const float *A, int lda, int K, const float *__restrict__ B, int ldb, int width, float *out,
                                        int ldo, int nout, const Epi &e, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < K; k0 += KC) {
        const int kc = min(KC, K - k0);
        __syncthreads();
        for (int i = tid; i < kc * 32; i += NT) {
            const int r = i >> 5, c4 = (i & 31) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c4 < width) v = __ldg(reinterpret_cast<const float4 *>(B + (size_t)(k0 + r) * ldb + c4));
            *reinterpret_cast<float4 *>(s.Wst + r * 128 + c4) = v;
        }
        __syncthreads();
        const float *a = A + (ty * 4) * lda + k0;
#pragma unroll 2
        for (int k = 0; k < kc; k += 4) {
            float4 av[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = *reinterpret_cast<const float4 *>(a + i * lda + k);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float4 b0 = *reinterpret_cast<const float4 *>(s.Wst + (k + kk) * 128 + tx * 4);
                const float4 b1 = *reinterpret_cast<const float4 *>(s.Wst + (k + kk) * 128 + 64 + tx * 4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
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
    __syncthreads();   // every read of A is done: out may be a buffer A was not, but the next GEMM may read what this one writes
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = ty * 4 + i;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4);
            if (n >= nout) continue;
            float v = acc[i][j];
            if (e.bias) v += e.bias[n];
            if (e.r1p) v = fmaf(e.r1p[p], e.r1w[n], v);
            if (e.relu) v = fmaxf(v, 0.f);
            if (e.mask && !(e.mask[p * e.ldm + n] > 0.f)) v = 0.f;
            if (e.add) v += out[p * ldo + n];
            out[p * ldo + n] = v;
        }
    }
    __syncthreads();
}

// Weight-gradient tile: part[n][c] += sum_p Y[p][n] * X[p][c] for n < nrows (<= 128), c < ncols (<= 128), p over the tile in order.
// Each element of `part` has one owner thread, so the read-modify-write needs no atomics.
__device__ __forceinline__ void gemm_w(const float *Y, int ldy, int nrows, const float *X, int ldx, int ncols, float *__restrict__ part, int ldp,
                                       int tid) {
    const int ty = tid >> 4, tx = tid & 15;
    const bool wide = ncols > 64;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
#pragma unroll 2
    for (int p = 0; p < TP; ++p) {
        const float4 a0 = *reinterpret_cast<const float4 *>(Y + p * ldy + ty * 4);
        const float4 a1 = *reinterpret_cast<const float4 *>(Y + p * ldy + 64 + ty * 4);
        const float4 b0 = *reinterpret_cast<const float4 *>(X + p * ldx + tx * 4);
        const float4 b1 = wide ? *reinterpret_cast<const float4 *>(X + p * ldx + 64 + tx * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int n = i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4);
        if (n >= nrows) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4);
            if (c < ncols) part[(size_t)n * ldp + c] += acc[i][j];
        }
    }
}

// Narrow layer forward: out[p][o] = sum_k A[p][k] * W[o][k], k < 128, o < NO; four threads per point, fixed reduction order.
template <int NO>
__device__ __forceinline__ void narrow_fwd(const float *A, int lda, const float *__restrict__ W, int no, int tid, float (&out)[NO]) {
    const int p = tid >> 2, q = tid & 3;
    const float *ar = A + p * lda + q * 32;
#pragma unroll
    for (int o = 0; o < NO; ++o) {
        float v = 0.f;
        if (o < no) {
            const float *wr = W + o * 128 + q * 32;
#pragma unroll 8
            for (int k = 0; k < 32; ++k) v = fmaf(ar[k], __ldg(wr + k), v);
        }
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        out[o] = v;
    }
}

// Narrow layer weight gradient: part[o][k] += sum_p g[p][o] * A[p][k], o < no, k < 128.
__device__ __forceinline__ void narrow_dw(const float *g, const float *A, int lda, int no, float *__restrict__ part, int tid) {
    for (int e = tid; e < no * 128; e += NT) {
        const int o = e >> 7, k = e & 127;
        float v = 0.f;
        for (int p = 0; p < TP; ++p) v = fmaf(g[p * 4 + o], A[p * lda + k], v);
        part[e] += v;
    }
}

// Narrow layer input gradient through a ReLU, in place: A[p][k] = A[p][k] > 0 ? sum_o g[p][o] * W[o][k] : 0.
__device__ __forceinline__ void narrow_dx_relu(const float *g, float *A, int lda, const float *__restrict__ W, int no, int tid) {
    for (int e = tid; e < TP * 128; e += NT) {
        const int p = e >> 7, k = e & 127;
        float v = 0.f;
        for (int o = 0; o < no; ++o) v = fmaf(g[p * 4 + o], __ldg(W + o * 128 + k), v);
        A[p * lda + k] = A[p * lda + k] > 0.f ? v : 0.f;
    }
}

// column sums over the tile: part[n] += sum_p Y[p][n]
__device__ __forceinline__ void colsum(const float *Y, int ldy, float *__restrict__ part, int tid) {
    if (tid < 128) {
        float v = 0.f;
        for (int p = 0; p < TP; ++p) v += Y[p * ldy + tid];
        part[tid] += v;
    }
}

// GridEncoder.forward's map to [0,1]: (x + bound) / (2 * bound) (grid.py:152)
__device__ __forceinline__ void to_unit(const float *x, float bound, int D, float *u) {
    const float twob = 2.0f * bound;
    for (int d = 0; d < D; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], bound), twob);
}

// ---- the forward of one tile; leaves B0 = [SH | geo], B1 = colour hidden, B2 = sigma hidden 2, PA = [pos | ambient] features ----
__device__ void tile_forward(const FieldArgs &a, Smem &s, uint32_t tile, int tid, bool write_out) {
    const uint32_t base = tile * TP;
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
    const int p = tid & (TP - 1), lg = tid >> 6;
    // position grid -> PA[:, 0:32]
    {
        float u[3];
        to_unit(s.pt + p * 4, a.bound, 3, u);
        for (int l = lg * 4; l < lg * 4 + 4; ++l) {
            const float2 f = s.valid[p] ? grid_lookup3(a.pos_gm, a.pos_tab, l, u[0], u[1], u[2]) : make_float2(0.f, 0.f);
            *reinterpret_cast<float2 *>(s.PA + p * LDPA + 2 * l) = f;
        }
    }
    // ambient net (conditioning folded into the first layer's bias) -> tanh
    Epi e;
    e.relu = true;
    e.bias = a.wt + FieldWt::bias_a0;
    gemm_pt(s, s.PA, LDPA, 32, a.wt + FieldWt::a0, 128, 128, s.B1, LD1, 128, e, tid);
    e.bias = nullptr;
    gemm_pt(s, s.B1, LD1, 128, a.wt + FieldWt::a1, 128, 128, s.B2, LD1, 128, e, tid);
    {
        float o[3];
        narrow_fwd<3>(s.B2, LD1, a.w[2], a.amb_dim, tid, o);
        if ((tid & 3) == 0) {
            const int q = tid >> 2;
            for (int d = 0; d < a.amb_dim; ++d) s.amb[q * 4 + d] = tanhf(o[d]);
        }
    }
    __syncthreads();
    // ambient grid (bound 1) -> PA[:, 32:64]
    {
        float u[3] = {0.f, 0.f, 0.f};
        for (int d = 0; d < a.amb_dim; ++d) u[d] = __fdiv_rn(__fadd_rn(s.amb[p * 4 + d], 1.0f), 2.0f);
        for (int l = lg * 4; l < lg * 4 + 4; ++l) {
            float2 f = make_float2(0.f, 0.f);
            if (s.valid[p]) f = a.amb_dim == 3 ? grid_lookup3(a.amb_gm, a.amb_tab, l, u[0], u[1], u[2]) : grid_lookup2(a.amb_gm, a.amb_tab, l, u[0], u[1]);
            *reinterpret_cast<float2 *>(s.PA + p * LDPA + 32 + 2 * l) = f;
        }
    }
    // sigma net
    gemm_pt(s, s.PA, LDPA, 64, a.wt + FieldWt::s0, 128, 128, s.B1, LD1, 128, e, tid);
    gemm_pt(s, s.B1, LD1, 128, a.wt + FieldWt::s1, 128, 128, s.B2, LD1, 128, e, tid);
    {
        float o[1];
        narrow_fwd<1>(s.B2, LD1, a.w[5], 1, tid, o);
        if ((tid & 3) == 0) s.h0[tid >> 2] = o[0];
    }
    e.relu = false;
    gemm_pt(s, s.B2, LD1, 128, a.wt + FieldWt::s2, 128, 128, s.B0 + 16, LD0, 128, e, tid);   // geo features -> B0[:, 16:144]
    if (tid < TP) {   // SH(dir) -> B0[:, 0:16]
        float sh[16];
        sh4(s.dr[tid * 4], s.dr[tid * 4 + 1], s.dr[tid * 4 + 2], sh);
        for (int j = 0; j < 16; ++j) s.B0[tid * LD0 + j] = sh[j];
    }
    // colour net (individual code folded into the first layer's bias) -> sigmoid
    e.relu = true;
    e.bias = a.wt + FieldWt::bias_c0;
    gemm_pt(s, s.B0, LD0, 144, a.wt + FieldWt::c0, 128, 128, s.B1, LD1, 128, e, tid);
    {
        float o[3];
        narrow_fwd<3>(s.B1, LD1, a.w[7], 3, tid, o);
        if ((tid & 3) == 0) {
            const int q = tid >> 2;
            for (int c = 0; c < 3; ++c) s.g3[q * 4 + c] = 1.0f / (1.0f + expf(-o[c]));
        }
    }
    __syncthreads();
    if (write_out && tid < TP && s.valid[tid]) {
        const size_t q = base + tid;
        a.sigma[q] = expf(s.h0[tid]);   // trunc_exp forward is plain exp (utils.py:36-41); density_scale is the caller's
        for (int c = 0; c < 3; ++c) a.color[q * 3 + c] = s.g3[tid * 4 + c];
        for (int d = 0; d < a.amb_dim; ++d) a.ambient[q * a.amb_dim + d] = s.amb[tid * 4 + d];
    }
    __syncthreads();
}

}  // namespace

// k-major transposes of the forward weight operands and the two folded biases (FieldWt), one thread per output float
__global__ void k_field_relayout(const __grid_constant__ FieldArgs a) {
    const uint32_t total = (uint32_t)FieldWt::total;
    const int ldc0 = 144 + a.ind_dim;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        float v;
        if (i >= FieldWt::bias_c0) {
            const uint32_t n = i - (uint32_t)FieldWt::bias_c0;
            v = 0.f;
            for (int j = 0; j < a.ind_dim; ++j) v = fmaf(a.code[j], a.w[6][n * ldc0 + 144 + j], v);
        } else if (i >= FieldWt::bias_a0) {
            const uint32_t n = i - (uint32_t)FieldWt::bias_a0;
            v = 0.f;
            for (int k = 0; k < 64; ++k) v = fmaf(a.cond[k], a.w[0][n * 96 + 32 + k], v);
        } else {
            const float *W;
            int ld, row0 = 0;
            uint32_t r;
            if (i >= FieldWt::c0) { W = a.w[6]; ld = ldc0; r = i - (uint32_t)FieldWt::c0; }
            else if (i >= FieldWt::s2) { W = a.w[5]; ld = 128; row0 = 1; r = i - (uint32_t)FieldWt::s2; }
            else if (i >= FieldWt::s1) { W = a.w[4]; ld = 128; r = i - (uint32_t)FieldWt::s1; }
            else if (i >= FieldWt::s0) { W = a.w[3]; ld = 64; r = i - (uint32_t)FieldWt::s0; }
            else if (i >= FieldWt::a1) { W = a.w[1]; ld = 128; r = i - (uint32_t)FieldWt::a1; }
            else { W = a.w[0]; ld = 96; r = i; }
            const uint32_t k = r >> 7, n = r & 127;
            v = W[(size_t)(row0 + n) * ld + k];
        }
        a.wt[i] = v;
    }
}

__global__ void __launch_bounds__(NT, 1) k_field_fwd(const __grid_constant__ FieldArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const uint32_t n_tiles = (a.M + TP - 1) / TP;
    for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) tile_forward(a, s, t, threadIdx.x, true);
}

// Backward of one tile after its forward (B0 = [SH | geo], B1 = c1, B2 = s2, PA = [pos | amb features]):
//   1 colour logits' gradient, dW c1;  2 g_c1 in place (B1);  3 dW c0, column sums;  4 g_geo = g_c1 W_c0[:, 16:144] -> B0
//   5 dW s2;  6 g_s2 -> B1;  7 s1 recomputed -> B0;  8 dW s1;  9 g_s1 -> B2;  10 dW s0;  11 g_[pos|amb feat] -> B0[:, 0:64]
//   12 ambient grid: table scatter, input gradient, tanh';  13 a1 -> B1, a2 -> B2 recomputed;  14 dW a2, g_a2 in place (B2)
//   15 dW a1;  16 g_a1 in place (B1), column sums, dW a0;  17 g_pos += g_a1 W_a0[:, 0:32];  18 position grid: table scatter
__global__ void __launch_bounds__(NT, 1) k_field_bwd(const __grid_constant__ FieldArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem &s = *reinterpret_cast<Smem *>(smem_raw);
    const int tid = threadIdx.x;
    float *part = a.part + (size_t)blockIdx.x * FieldPart::total;
    for (size_t i = tid; i < FieldPart::total; i += NT) part[i] = 0.f;
    __syncthreads();
    const uint32_t n_tiles = (a.M + TP - 1) / TP;
    const uint32_t t0 = (uint32_t)((uint64_t)n_tiles * blockIdx.x / gridDim.x), t1 = (uint32_t)((uint64_t)n_tiles * (blockIdx.x + 1) / gridDim.x);
    const int p = tid & (TP - 1), lg = tid >> 6;
    for (uint32_t t = t0; t < t1; ++t) {
        tile_forward(a, s, t, tid, false);
        const uint32_t base = t * TP;
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
        narrow_dw(s.g3, s.B1, LD1, 3, part + FieldPart::c1, tid);
        __syncthreads();
        // 2
        narrow_dx_relu(s.g3, s.B1, LD1, a.w[7], 3, tid);
        __syncthreads();
        // 3
        colsum(s.B1, LD1, part + FieldPart::csc, tid);
        gemm_w(s.B1, LD1, 128, s.B0, LD0, 128, part + FieldPart::c0, 144, tid);
        gemm_w(s.B1, LD1, 128, s.B0 + 128, LD0, 16, part + FieldPart::c0 + 128, 144, tid);
        // 4
        Epi e;
        gemm_pt(s, s.B1, LD1, 128, a.w[6] + 16, 144 + a.ind_dim, 128, s.B0, LD0, 128, e, tid);
        // 5: the sigma row, then the geo rows
        if (tid < 128) {
            const int k = tid;
            float v = 0.f;
            for (int q = 0; q < TP; ++q) v = fmaf(s.gh0[q], s.B2[q * LD1 + k], v);
            part[FieldPart::s2 + k] += v;
        }
        gemm_w(s.B0, LD0, 128, s.B2, LD1, 128, part + FieldPart::s2 + 128, 128, tid);
        // 6: g_s2 = (g_geo W_s2[1:129] + g_h0 W_s2[0]) masked by s2 > 0
        e.r1p = s.gh0; e.r1w = a.w[5]; e.mask = s.B2; e.ldm = LD1;
        gemm_pt(s, s.B0, LD0, 128, a.w[5] + 128, 128, 128, s.B1, LD1, 128, e, tid);
        // 7
        e = Epi();
        e.relu = true;
        gemm_pt(s, s.PA, LDPA, 64, a.wt + FieldWt::s0, 128, 128, s.B0, LD0, 128, e, tid);
        // 8
        gemm_w(s.B1, LD1, 128, s.B0, LD0, 128, part + FieldPart::s1, 128, tid);
        // 9
        e = Epi();
        e.mask = s.B0; e.ldm = LD0;
        gemm_pt(s, s.B1, LD1, 128, a.w[4], 128, 128, s.B2, LD1, 128, e, tid);
        // 10
        gemm_w(s.B2, LD1, 128, s.PA, LDPA, 64, part + FieldPart::s0, 64, tid);
        // 11
        e = Epi();
        gemm_pt(s, s.B2, LD1, 128, a.w[3], 64, 64, s.B0, LD0, 64, e, tid);
        // 12: ambient grid -- table gradient, input gradient through dy_dx, (x+1)/2 and tanh'
        {
            float u[3] = {0.f, 0.f, 0.f};
            for (int d = 0; d < a.amb_dim; ++d) u[d] = __fdiv_rn(__fadd_rn(s.amb[p * 4 + d], 1.0f), 2.0f);
            float gin[3] = {0.f, 0.f, 0.f};
            if (s.valid[p]) {
                for (int l = lg * 4; l < lg * 4 + 4; ++l) {
                    const float2 g = *reinterpret_cast<const float2 *>(s.B0 + p * LD0 + 32 + 2 * l);
                    if (a.amb_dim == 3) {
                        grid_scatter<3>(a.amb_gm, l, u, g, a.g_amb_tab);
                        grid_input_grad<3>(a.amb_gm, a.amb_tab, l, u, g, gin);
                    } else {
                        grid_scatter<2>(a.amb_gm, l, u, g, a.g_amb_tab);
                        grid_input_grad<2>(a.amb_gm, a.amb_tab, l, u, g, gin);
                    }
                }
            }
            for (int d = 0; d < 3; ++d) s.gu[(lg * TP + p) * 4 + d] = gin[d];
        }
        __syncthreads();
        if (tid < TP) {
            const bool v = s.valid[tid] != 0;
            for (int d = 0; d < 3; ++d) {
                float g = 0.f;
                if (v && d < a.amb_dim) {
                    // sum over levels in level order (levels 4j..4j+3 in group j), then the (x + 1) / 2 map's 1/2
                    const float gl = ((s.gu[(0 * TP + tid) * 4 + d] + s.gu[(1 * TP + tid) * 4 + d]) + s.gu[(2 * TP + tid) * 4 + d]) +
                                     s.gu[(3 * TP + tid) * 4 + d];
                    const float y = s.amb[tid * 4 + d];
                    g = (gl / 2.0f + a.g_ambient[(size_t)(base + tid) * a.amb_dim + d]) * (1.0f - y * y);
                }
                s.g3[tid * 4 + d] = g;
            }
        }
        // 13
        e = Epi();
        e.relu = true;
        e.bias = a.wt + FieldWt::bias_a0;
        gemm_pt(s, s.PA, LDPA, 32, a.wt + FieldWt::a0, 128, 128, s.B1, LD1, 128, e, tid);
        e.bias = nullptr;
        gemm_pt(s, s.B1, LD1, 128, a.wt + FieldWt::a1, 128, 128, s.B2, LD1, 128, e, tid);
        // 14
        narrow_dw(s.g3, s.B2, LD1, a.amb_dim, part + FieldPart::a2, tid);
        __syncthreads();
        narrow_dx_relu(s.g3, s.B2, LD1, a.w[2], a.amb_dim, tid);
        __syncthreads();
        // 15
        gemm_w(s.B2, LD1, 128, s.B1, LD1, 128, part + FieldPart::a1, 128, tid);
        // 16
        e = Epi();
        e.mask = s.B1; e.ldm = LD1;
        gemm_pt(s, s.B2, LD1, 128, a.w[1], 128, 128, s.B1, LD1, 128, e, tid);
        colsum(s.B1, LD1, part + FieldPart::csa, tid);
        gemm_w(s.B1, LD1, 128, s.PA, LDPA, 32, part + FieldPart::a0, 32, tid);
        // 17
        e = Epi();
        e.add = true;
        gemm_pt(s, s.B1, LD1, 128, a.w[0], 96, 32, s.B0, LD0, 32, e, tid);
        // 18: position grid -- table gradient only (xyzs never requires grad in the reference)
        if (s.valid[p]) {
            float u[3];
            to_unit(s.pt + p * 4, a.bound, 3, u);
            for (int l = lg * 4; l < lg * 4 + 4; ++l)
                grid_scatter<3>(a.pos_gm, l, u, *reinterpret_cast<const float2 *>(s.B0 + p * LD0 + 2 * l), a.g_pos_tab);
        }
        __syncthreads();
    }
}

// Sums the per-CTA partials in CTA order into the caller's gradient buffers; the conditioning / code columns and the input gradients
// of cond_feat and the individual code follow from the column sums.  blockIdx.y selects the output.
__global__ void k_field_reduce(const __grid_constant__ FieldArgs a) {
    const int seg = blockIdx.y;
    const uint32_t G = a.n_cta;
    const size_t P = FieldPart::total;
    auto sum = [&](size_t off) {
        float v = 0.f;
        for (uint32_t c = 0; c < G; ++c) v += a.part[c * P + off];
        return v;
    };
    const int ldc0 = 144 + a.ind_dim;
    uint32_t n_out;
    switch (seg) {
        case 0: n_out = 128 * 96; break;
        case 1: n_out = 128 * 128; break;
        case 2: n_out = (uint32_t)a.amb_dim * 128; break;
        case 3: n_out = 128 * 64; break;
        case 4: n_out = 128 * 128; break;
        case 5: n_out = 129 * 128; break;
        case 6: n_out = 128 * (uint32_t)ldc0; break;
        case 7: n_out = 3 * 128; break;
        case 8: n_out = 64; break;
        default: n_out = (uint32_t)a.ind_dim; break;
    }
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += gridDim.x * blockDim.x) {
        float v;
        switch (seg) {
            case 0: {
                const uint32_t n = i / 96, k = i % 96;
                v = k < 32 ? sum(FieldPart::a0 + n * 32 + k) : sum(FieldPart::csa + n) * a.cond[k - 32];
                break;
            }
            case 1: v = sum(FieldPart::a1 + i); break;
            case 2: v = sum(FieldPart::a2 + i); break;
            case 3: v = sum(FieldPart::s0 + i); break;
            case 4: v = sum(FieldPart::s1 + i); break;
            case 5: v = sum(FieldPart::s2 + i); break;
            case 6: {
                const uint32_t n = i / ldc0, k = i % ldc0;
                v = k < 144 ? sum(FieldPart::c0 + n * 144 + k) : sum(FieldPart::csc + n) * a.code[k - 144];
                break;
            }
            case 7: v = sum(FieldPart::c1 + i); break;
            case 8: {
                v = 0.f;
                for (int n = 0; n < 128; ++n) v = fmaf(sum(FieldPart::csa + n), a.w[0][n * 96 + 32 + i], v);
                break;
            }
            default: {
                v = 0.f;
                for (int n = 0; n < 128; ++n) v = fmaf(sum(FieldPart::csc + n), a.w[6][n * ldc0 + 144 + i], v);
                break;
            }
        }
        if (seg < 8) a.g_w[seg][i] = v;
        else if (seg == 8) a.g_cond[i] = v;
        else a.g_code[i] = v;
    }
}

cudaError_t launch_field_relayout(const FieldArgs &a, cudaStream_t st) {
    k_field_relayout<<<grid_for(FieldWt::total, 256), 256, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_field_fwd(const FieldArgs &a, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(k_field_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    const uint32_t n_tiles = (a.M + TP - 1) / TP;
    const int blocks = (int)(n_tiles < (uint32_t)sm_count() ? n_tiles : (uint32_t)sm_count());
    k_field_fwd<<<blocks, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_field_bwd(const FieldArgs &a, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(k_field_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    k_field_bwd<<<a.n_cta, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_field_reduce(const FieldArgs &a, cudaStream_t st) {
    k_field_reduce<<<dim3(64, 10), 256, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gfpp
