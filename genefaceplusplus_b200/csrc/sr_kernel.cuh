// sr_kernel.cuh -- argument blocks of the super-resolution head kernels (see sr_kernel.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gfpp {

// One implicit-GEMM convolution layer on wgmma (k_sr_conv<LAYER>):
//   LAYER 0: block0.conv1  128 -> 128, 3x3, at HxW            (+ toRGB, + rgb skip -> img0)
//   LAYER 1: block1.conv0  128 -> 64,  3x3 transposed stride 2 + FIR, merged into four 3x3 phase kernels: HxW -> 2Hx2W
//   LAYER 2: block1.conv1   64 -> 64,  3x3, at HxW (= 512)    (+ toRGB, + 2x FIR up-sampled skip -> final image)
struct SrConvArgs {
    const __half *in;          // NHWC fp16 [F, H, W, CIN]
    int F, H, W;               // input (= GEMM row) grid; W % 128 == 0
    const unsigned char *wt;   // weight chunks in streaming order: chunk c = (tap, 64-channel block), N-blocks inside a chunk
    const float *bias;         // [COUT]
    const float *noise;        // [H_out * W_out] (+ f * noise_fstride), already multiplied by noise_strength; or nullptr
    long long noise_fstride;   // 0: one plane for every frame (noise_mode 'const'); H_out*W_out: one per frame ('random')
    __half *out;               // LAYER 0: [F,H,W,128]; LAYER 1: [F,2H,2W,64]; LAYER 2: [F,H,W,64] for the backward, or nullptr
    const float *rgb_w;        // [3][COUT] effective toRGB weights (layers 0 and 2)
    const float *rgb_b;        // [3]
    const float *img_in;       // LAYER 0: the NeRF image [F,H,W,3]; LAYER 2: img0 [F,H/2,W/2,3]
    float *img_out;            // LAYER 0: img0 [F,H,W,3]; LAYER 2: the final image [F,3,H,W] (planar), or nullptr with img_u8
    int clamp01;               // LAYER 2: clamp the final image to [0,1] (what every caller of the SR head does next)
    unsigned char *img_u8;     // LAYER 2: optional video frames [F,H,W,3] (interleaved) = (int)(clamp01(rgb) * 255); else nullptr
};

// block0.conv0: 3 -> 128, 3x3, fp32 on CUDA cores (K = 27 is no tensor-core shape), fp16 NHWC out
struct SrConvInArgs {
    const float *in;           // [F, H, W, 3] fp32 (the renderer's rgb_map)
    int F, H, W;
    const float *w;            // [27][128] k-major, k = (ky*3+kx)*3 + ci
    const float *bias;         // [128]
    const float *noise;
    long long noise_fstride;
    __half *out;               // [F, H, W, 128]
};

constexpr int SR_TILE_ROWS = 128;                    // GEMM rows (pixels of one image row) per tile
constexpr int sr_layer_cin(int layer) { return layer == 2 ? 64 : 128; }
constexpr int sr_layer_nb(int layer) { return layer == 1 ? 2 : 1; }        // N-blocks (weight tiles per K chunk)
constexpr int sr_layer_nrows(int layer) { return layer == 2 ? 64 : 128; }  // rows (= MMA N) of one weight tile
constexpr int sr_layer_nchunk(int layer) { return 9 * sr_layer_cin(layer) / 64; }
constexpr int sr_layer_chunk_bytes(int layer) { return sr_layer_nb(layer) * sr_layer_nrows(layer) * 128; }
constexpr int sr_layer_weight_bytes(int layer) { return sr_layer_nchunk(layer) * sr_layer_chunk_bytes(layer); }

cudaError_t launch_sr_conv_in(const SrConvInArgs &a, cudaStream_t st);
cudaError_t launch_sr_conv(int layer, const SrConvArgs &a, cudaStream_t st);

}  // namespace gfpp
