// tc.cuh -- Hopper tensor-core (wgmma) building blocks for the tiny-MLP GEMMs and the SR convolutions, sm_90a.
//
// D[64 x N] (fp32, registers of one warpgroup) (+)= A[64 x K] (smem, K-major) * W[N x K]^T (smem, K-major), 16-bit
// operands (fp16 or bf16), issued by the 128 threads of a warpgroup (wgmma.mma_async), completion awaited with
// wgmma.commit_group / wait_group.  nn.Linear weights are [out, in] = [N, K] row-major, i.e. already K-major.
// A 128-row operand tile is two M = 64 halves: half h starts 64 rows (8 KB of an SW128 tile, 2 KB of a K16 tile) further.
//
// Operand tiles in shared memory use the canonical GMMA K-major layouts:
//   * SW128 tile: [rows x 64 elements], 128-byte rows, 8-row groups of 1024 B (SBO), 16-byte chunks XOR-swizzled
//     with the row index (Swizzle<3,4,3>); tile base 1024-byte aligned.
//   * K16 tile (no swizzle / "interleave"): [rows x 16 elements] as 8x16B core matrices: the two K-chunks of a
//     group are 128 B apart (LBO), groups are 256 B apart (SBO).
// Accumulator fragment of m64nNk16: register i of lane l in warp w (0..3) of the warpgroup holds row
// 16w + l/4 + 8*((i>>1)&1), column 8*(i>>2) + 2*(l%4) + (i&1)  (frag_row / frag_col below).
// "split" precision: x = hi + lo with hi = rn16(x), lo = rn16(x - hi); A*W ~= Ah*Wh + Ah*Wl + Al*Wh accumulated
// in the same fp32 accumulator (3 MMAs per k-step) -- bf16x3 gives ~16 mantissa bits.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gfpp {
namespace tc {

// FP16_ROBUST: fp16 operands, hi/lo split (3 MMAs per k-step) on the AMBIENT net only + 16-bit fixed-point position table:
// the two places whose rounding the field amplifies (tools/error_budget.py); everything else single fp16 images.
enum Precision : int { FP32_SIMT = 0, FP16_X1 = 1, BF16_X3 = 2, BF16_X1 = 3, FP16_ROBUST = 4 };

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier / bulk copy (shared with head_kernel.cu) ----
__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
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
// plain arrive (count 1) by the executing thread; release semantics at CTA scope
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (tensor core / TMA reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// one lane of a converged warp
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
// barrier of the 128 threads of one warpgroup (named barrier `id` > 0; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// ---- descriptors ----
// shared-memory matrix descriptor (GMMA), SW128 K-major: SBO = 1024 B, LBO unused (=1), layout type 1 (128-byte swizzle)
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// no-swizzle K-major, K = 16 elements: LBO = 128 B (between the two 16-byte K chunks), SBO = 256 B (8-row groups)
__device__ __forceinline__ uint64_t desc_k16(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}
// byte offset of M-half `h` (rows 64h..64h+63) inside a 128-row operand tile
constexpr uint32_t SW128_HALF = 8192, K16_HALF = 2048;

// ---- wgmma (warpgroup-collective: all 128 threads, converged) ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the compiler from moving accumulator reads / writes across the asynchronous MMA window
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void acc_zero(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) d[i] = 0.f;
}
__device__ __forceinline__ int frag_row(int i, int lane, int wwarp) { return 16 * wwarp + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }

// D[64 x N] (+)= A * W^T, one k-step of 16; `acc` = 0: D = A * W^T
template <int N, bool BF16>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc);
#define GFPP_ACC8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define GFPP_WGMMA_N16(TY) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}" \
                 : GFPP_ACC8(0) : "l"(da), "l"(db), "r"(acc))
template <> __device__ __forceinline__ void wgmma<16, false>(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N16("f16"); }
template <> __device__ __forceinline__ void wgmma<16, true>(float (&d)[8], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N16("bf16"); }
#undef GFPP_WGMMA_N16
#define GFPP_WGMMA_N64(TY) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}" \
                 : GFPP_ACC8(0), GFPP_ACC8(8), GFPP_ACC8(16), GFPP_ACC8(24) : "l"(da), "l"(db), "r"(acc))
template <> __device__ __forceinline__ void wgmma<64, false>(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N64("f16"); }
template <> __device__ __forceinline__ void wgmma<64, true>(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N64("bf16"); }
#undef GFPP_WGMMA_N64
#define GFPP_WGMMA_N128(TY) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}" \
                 : GFPP_ACC8(0), GFPP_ACC8(8), GFPP_ACC8(16), GFPP_ACC8(24), GFPP_ACC8(32), GFPP_ACC8(40), GFPP_ACC8(48), GFPP_ACC8(56) : "l"(da), "l"(db), "r"(acc))
template <> __device__ __forceinline__ void wgmma<128, false>(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N128("f16"); }
template <> __device__ __forceinline__ void wgmma<128, true>(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N128("bf16"); }
#undef GFPP_WGMMA_N128
#define GFPP_WGMMA_N144(TY) \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\twgmma.mma_async.sync.aligned.m64n144k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, p, 1, 1, 0, 0;\n\t}" \
                 : GFPP_ACC8(0), GFPP_ACC8(8), GFPP_ACC8(16), GFPP_ACC8(24), GFPP_ACC8(32), GFPP_ACC8(40), GFPP_ACC8(48), GFPP_ACC8(56), GFPP_ACC8(64) : "l"(da), "l"(db), "r"(acc))
template <> __device__ __forceinline__ void wgmma<144, false>(float (&d)[72], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N144("f16"); }
template <> __device__ __forceinline__ void wgmma<144, true>(float (&d)[72], uint64_t da, uint64_t db, uint32_t acc) { GFPP_WGMMA_N144("bf16"); }
#undef GFPP_WGMMA_N144
#undef GFPP_ACC8
// ---- warp-level mma.sync (one warp, operands in registers) ----
// D[16 x 8] += A[16 x 16] * B[16 x 8], fp16 operands, fp32 accumulation.  Lane l = 4g + t holds A rows g (a0, a2) and g + 8
// (a1, a3) at K columns 2t, 2t + 1 (a0, a1) and 2t + 8, 2t + 9 (a2, a3); B K rows 2t, 2t + 1 (b0) and 2t + 8, 2t + 9 (b1) of
// column g; C/D rows g (c0, c1) and g + 8 (c2, c3) at columns 2t, 2t + 1.  The 16 columns 16kb .. 16kb + 15 of a warp's m64
// accumulator fragment are this A fragment as they stand: a_j = the pair (d[8kb + 2j], d[8kb + 2j + 1]).
__device__ __forceinline__ void mma_m16n8k16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// all k-steps of one SW128 K-tile (ksteps x 16 elements); `acc_first` = 0 starts a new accumulation
template <int N, bool BF16>
__device__ __forceinline__ void wgmma_sw(float (&d)[N / 2], uint32_t a, uint32_t w, int ksteps, uint32_t acc_first) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (k < ksteps) wgmma<N, BF16>(d, desc_sw128(a + (uint32_t)k * 32u), desc_sw128(w + (uint32_t)k * 32u), (k > 0) ? 1u : acc_first);
}

// ---- operand tile addressing (byte offsets inside a tile) ----
__host__ __device__ __forceinline__ uint32_t sw128_off(int row, int chunk /*16B chunk 0..7*/) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}
__host__ __device__ __forceinline__ uint32_t k16_off(int row, int chunk /*0..1*/) {
    return (uint32_t)((row >> 3) * 256 + chunk * 128 + (row & 7) * 16);
}

// ---- 16-bit conversion with optional hi/lo split ----
template <bool BF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    if (BF16) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&h);
    } else {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&h);
    }
}
template <bool BF16>
__device__ __forceinline__ float round16(float a) {
    if (BF16) return __bfloat162float(__float2bfloat16_rn(a));
    return __half2float(__float2half_rn(a));
}
// 8 consecutive K values -> one 16-byte chunk of the hi tile (and of the lo tile when SPLIT)
template <bool BF16, bool SPLIT>
__device__ __forceinline__ void store_chunk(unsigned char *hi_tile, unsigned char *lo_tile, uint32_t off, const float *v) {
    uint4 h;
    h.x = pack2<BF16>(v[0], v[1]); h.y = pack2<BF16>(v[2], v[3]); h.z = pack2<BF16>(v[4], v[5]); h.w = pack2<BF16>(v[6], v[7]);
    *reinterpret_cast<uint4 *>(hi_tile + off) = h;
    if (SPLIT) {
        float r[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) r[i] = v[i] - round16<BF16>(v[i]);
        uint4 l;
        l.x = pack2<BF16>(r[0], r[1]); l.y = pack2<BF16>(r[2], r[3]); l.z = pack2<BF16>(r[4], r[5]); l.w = pack2<BF16>(r[6], r[7]);
        *reinterpret_cast<uint4 *>(lo_tile + off) = l;
    }
}
// two consecutive K values (an accumulator pair) -> 4 bytes of the hi tile (and of the lo tile when SPLIT) at column `col`
// of row `row` of an SW128 tile
template <bool BF16, bool SPLIT>
__device__ __forceinline__ void store_pair(unsigned char *hi_tile, unsigned char *lo_tile, int row, int col, float a, float b) {
    const uint32_t off = sw128_off(row, col >> 3) + (uint32_t)(col & 7) * 2u;
    *reinterpret_cast<uint32_t *>(hi_tile + off) = pack2<BF16>(a, b);
    if (SPLIT) *reinterpret_cast<uint32_t *>(lo_tile + off) = pack2<BF16>(a - round16<BF16>(a), b - round16<BF16>(b));
}
// four 8x8 matrices of 16-bit pairs, one warp: lane l gives the shared address of row l%8 of matrix l/8 (16 contiguous bytes), and
// register j holds the pair at row l/4, columns 2*(l%4) .. +1 of matrix j -- the layout of an accumulator fragment's pairs
__device__ __forceinline__ void stmatrix_x4(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}

// the inverse of stmatrix_x4: register j of lane l <- the pair at row l/4, columns 2*(l%4) .. +1 of matrix j (lane l addresses row
// l%8 of matrix l/8)
__device__ __forceinline__ void ldmatrix_x4(uint32_t saddr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(saddr)
                 : "memory");
}

// ---- transposed (MN-major) operands: D[64 x N] (+)= A^T * B with A [K x 64] and B [K x N] both row-major over K ----
// A [rows x 64 elements] SW128 tile read along its rows is the canonical MN-major SW128 layout as it stands: one 128-byte row per
// k, 8-row groups 1024 B apart (SBO), 64-element blocks of the M / N extent `lbo` bytes apart (LBO; unused when the extent is 64).
// A k-step of 16 is 16 rows: 2048 B.  This is the weight-gradient product dW = dY^T X with both operands point-major.
__device__ __forceinline__ uint64_t desc_sw128_mn(uint32_t saddr, uint32_t lbo) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
template <int N>
__device__ __forceinline__ void wgmma_tn(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc);
#define GFPP_ACC8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <> __device__ __forceinline__ void wgmma_tn<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n\t}"
                 : GFPP_ACC8(0), GFPP_ACC8(8), GFPP_ACC8(16), GFPP_ACC8(24) : "l"(da), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_tn<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n\t}"
                 : GFPP_ACC8(0), GFPP_ACC8(8), GFPP_ACC8(16), GFPP_ACC8(24), GFPP_ACC8(32), GFPP_ACC8(40), GFPP_ACC8(48), GFPP_ACC8(56) : "l"(da), "l"(db), "r"(acc));
}
#undef GFPP_ACC8

// ---- tf32 operands: D[64 x N] (+)= A[64 x 8] * W[N x 8]^T, one k-step of 8 (32 bytes of each row) ----
// W (smem, K-major) as no-swizzle K8 blocks: a k-step of 4-byte elements has the byte geometry of a K16 tile of 2-byte
// elements (two 16-byte K chunks 128 B apart, 8-row groups 256 B apart), so one block of N rows is N * 32 bytes and element
// (n, k) sits at k16_off(n, k / 4) + 4 * (k % 4).  Unlike SW128, a K extent of 48 or 80 needs no padding to 32-element rows.
// A comes from registers (tf32 is the one 4-byte type wgmma accepts there): lane l of warp w holds rows 16w + l/4 (a0, a2)
// and 16w + l/4 + 8 (a1, a3), K columns l%4 (a0, a1) and l%4 + 4 (a2, a3).  Values are tf32 bit patterns (rna_tf32).
__device__ __forceinline__ uint64_t desc_tf32_k8(uint32_t saddr) { return desc_k16(saddr); }
__device__ __forceinline__ uint32_t rna_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t acc);
#define GFPP_ACC8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <> __device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
                 : GFPP_ACC8(0), GFPP_ACC8(8) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
                 : GFPP_ACC8(0), GFPP_ACC8(8), GFPP_ACC8(16), GFPP_ACC8(24) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}
#undef GFPP_ACC8
// split tf32 over K steps: D = A_lo W_hi + A_hi W_lo + A_hi W_hi (the small products first), fp32 accumulation.
// W_hi / W_lo: K8 blocks of N rows, block j at + j * N * 32 bytes.  `acc_first` = 0 starts a new accumulation.  Issues and
// commits one group; the caller waits.
template <int N, int KS>
__device__ __forceinline__ void wgmma_tf32x3(float (&d)[N / 2], const uint32_t (&ahi)[KS][4], const uint32_t (&alo)[KS][4],
                                             uint32_t w_hi, uint32_t w_lo, uint32_t acc_first) {
    wg_fence();
#pragma unroll
    for (int j = 0; j < KS; ++j) wgmma_tf32<N>(d, alo[j], desc_tf32_k8(w_hi + (uint32_t)(j * N * 32)), j > 0 ? 1u : acc_first);
#pragma unroll
    for (int j = 0; j < KS; ++j) wgmma_tf32<N>(d, ahi[j], desc_tf32_k8(w_lo + (uint32_t)(j * N * 32)), 1u);
#pragma unroll
    for (int j = 0; j < KS; ++j) wgmma_tf32<N>(d, ahi[j], desc_tf32_k8(w_hi + (uint32_t)(j * N * 32)), 1u);
    wg_commit();
}

}  // namespace tc
}  // namespace gfpp
