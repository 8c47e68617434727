// video_kernels.cu -- uint8 RGB video frames to planar I420 (include/gfpp.h section N), sm_90a.
//
// The renderer's uint8 frames (k_epilogue's rgb_u8, the SR head's video output) are interleaved RGB [F,H,W,3]; video encoders
// take yuv420p.  One thread converts a block of BX columns x 2 rows: BX luma bytes per row and BX/2 bytes of each chroma plane.
// Frames are contiguous, so the input's rows 2g and 2g+1 form row pair g of the whole batch, and frame g / (H/2) owns it.
//   * BX = 4 (vector): three 32-bit loads per row, one 32-bit luma store per row and one 16-bit store per chroma plane.  Needs
//     W % 4 == 0 and both buffers 4-byte aligned, which make every row, plane and frame start 4-byte aligned (H*W % 8 == 0).
//   * BX = 2 (bytes): any even W and any alignment.
// Integer arithmetic only (BT.601 limited range, gfpp.h (N)), so every byte is reproducible on the host.
#include "launch.cuh"
#include "ops.cuh"

namespace gfpp {

namespace {

constexpr int I420_NT = 256;

__device__ __forceinline__ uint32_t i420_luma(uint32_t r, uint32_t g, uint32_t b) { return ((66u * r + 129u * g + 25u * b + 128u) >> 8) + 16u; }

// s*: the 2x2 block's channel sums; the shifts of negative values are arithmetic (floor), as in the header's formula
__device__ __forceinline__ void i420_chroma(int sr, int sg, int sb, uint32_t &u, uint32_t &v) {
    const int r = (sr + 2) >> 2, g = (sg + 2) >> 2, b = (sb + 2) >> 2;
    u = (uint32_t)(((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128);
    v = (uint32_t)(((112 * r - 94 * g - 18 * b + 128) >> 8) + 128);
}

template <int BX>
__device__ __forceinline__ void i420_load_row(const uint8_t *__restrict__ src, uint32_t (&p)[3 * BX]) {
    if constexpr (BX == 4) {
        const uint32_t *q = reinterpret_cast<const uint32_t *>(src);
#pragma unroll
        for (int w = 0; w < 3; ++w) {
            const uint32_t x = __ldg(q + w);
#pragma unroll
            for (int k = 0; k < 4; ++k) p[4 * w + k] = (x >> (8 * k)) & 0xffu;
        }
    } else {
#pragma unroll
        for (int k = 0; k < 3 * BX; ++k) p[k] = __ldg(src + k);
    }
}

template <int BX>
__global__ void __launch_bounds__(I420_NT) k_rgb_u8_to_i420(const uint8_t *__restrict__ rgb, uint64_t n_items, uint32_t W, uint32_t half_h,
                                                            uint8_t *__restrict__ out) {
    const uint32_t nb = W / BX;                               // thread blocks per row pair
    const uint64_t plane = 2ull * half_h * W;                 // H*W: luma bytes of a frame
    const uint64_t frame = plane + plane / 2;                 // H*W*3/2
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_items; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = i / nb;
        const uint32_t x = (uint32_t)(i - g * nb) * BX;
        const uint64_t f = g / half_h;
        const uint32_t j = (uint32_t)(g - f * half_h);
        const uint8_t *r0 = rgb + (2 * g * W + x) * 3;
        uint32_t p0[3 * BX], p1[3 * BX];
        i420_load_row<BX>(r0, p0);
        i420_load_row<BX>(r0 + 3ull * W, p1);
        uint32_t y0 = 0, y1 = 0, u = 0, v = 0;
#pragma unroll
        for (int k = 0; k < BX; ++k) {
            y0 |= i420_luma(p0[3 * k], p0[3 * k + 1], p0[3 * k + 2]) << (8 * k);
            y1 |= i420_luma(p1[3 * k], p1[3 * k + 1], p1[3 * k + 2]) << (8 * k);
        }
#pragma unroll
        for (int c = 0; c < BX / 2; ++c) {
            const int a = 6 * c;
            uint32_t uc, vc;
            i420_chroma((int)(p0[a] + p0[a + 3] + p1[a] + p1[a + 3]), (int)(p0[a + 1] + p0[a + 4] + p1[a + 1] + p1[a + 4]),
                        (int)(p0[a + 2] + p0[a + 5] + p1[a + 2] + p1[a + 5]), uc, vc);
            u |= uc << (8 * c);
            v |= vc << (8 * c);
        }
        uint8_t *yp = out + f * frame + 2ull * j * W + x;
        uint8_t *up = out + f * frame + plane + (uint64_t)j * (W / 2) + x / 2;
        uint8_t *vp = up + plane / 4;
        if constexpr (BX == 4) {
            *reinterpret_cast<uint32_t *>(yp) = y0;
            *reinterpret_cast<uint32_t *>(yp + W) = y1;
            *reinterpret_cast<uint16_t *>(up) = (uint16_t)u;
            *reinterpret_cast<uint16_t *>(vp) = (uint16_t)v;
        } else {
            yp[0] = (uint8_t)y0;
            yp[1] = (uint8_t)(y0 >> 8);
            yp[W] = (uint8_t)y1;
            yp[W + 1] = (uint8_t)(y1 >> 8);
            *up = (uint8_t)u;
            *vp = (uint8_t)v;
        }
    }
}

}  // namespace

// F, H, W validated by the caller: H and W even and non-zero, F * H * W * 3 representable
cudaError_t launch_rgb_u8_to_i420(const uint8_t *rgb, uint32_t F, uint32_t H, uint32_t W, uint8_t *out, cudaStream_t st) {
    const bool vec = W % 4 == 0 && (((uintptr_t)rgb | (uintptr_t)out) & 3u) == 0;
    const uint64_t pairs = (uint64_t)F * (H / 2);
    if (vec) {
        const uint64_t n = pairs * (W / 4);
        k_rgb_u8_to_i420<4><<<grid_for(n, I420_NT), I420_NT, 0, st>>>(rgb, n, W, H / 2, out);
    } else {
        const uint64_t n = pairs * (W / 2);
        k_rgb_u8_to_i420<2><<<grid_for(n, I420_NT), I420_NT, 0, st>>>(rgb, n, W, H / 2, out);
    }
    return cudaGetLastError();
}

}  // namespace gfpp
