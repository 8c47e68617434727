// sr_train_kernel.cuh -- argument blocks of the super-resolution head's backward (see sr_train_kernel.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gfpp {

// dgrad of one tensor-core layer of the SR head as a forward-shaped implicit GEMM on TF32 wgmma (k_srb_dgrad<MODE>):
//   MODE 0: block1.conv1   gradient [F,2R,2R,64]  -> [F,2R,2R,64],  times y'(x1a)
//   MODE 1: block1.conv0   gradient [F,2R,2R,64] read as the four output phases of the R grid (K = 9 x 256) -> [F,R,R,128],
//           plus toRGB0's adjoint of g_r0, times y'(x0b)
//   MODE 2: block0.conv1   gradient [F,R,R,128]  -> [F,R,R,128],    times y'(x0a)
struct SrDgradArgs {
    const float *g;            // gradient w.r.t. the layer's pre-activation output, fp32 NHWC
    int F, H, W;               // GEMM grid (the layer's input grid); W % 128 == 0
    const unsigned char *wt;   // dgrad weight image (sr_dgrad_weight_bytes): tf32 K8 blocks in streaming order
    const __half *act;         // [F,H,W,N] the stored activation whose derivative the epilogue applies
    const float *rgb_w;        // MODE 1: toRGB0 weights [3][128]
    const float *g_rgb;        // MODE 1: gradient of toRGB0's output [F,H,W,3] (after its clamp)
    float *out;                // [F,H,W,N]
};

// wgrad of one tensor-core layer: partial[s][m][tap * CI + ci] = sum over the pixels of slice s of g[p, m] x[p + tap, ci]
//   MODE 0: block1.conv1  (m < 64,  x = x1a at 2R, CI = 64)
//   MODE 1: block1.conv0  (m = phase * 64 + co < 256, g read from the 2R grid at the phase's pixel, x = x0b at R, CI = 128)
//   MODE 2: block0.conv1  (m < 128, x = x0a at R, CI = 128)
struct SrWgradArgs {
    const float *g;
    const __half *x;
    int F, H, W;               // the grid of x; W % 128 == 0
    int slices;
    float *partial;
};

constexpr int sr_dgrad_cg(int mode) { return mode == 0 ? 64 : mode == 1 ? 256 : 128; }   // K channels per tap
constexpr int sr_dgrad_n(int mode) { return mode == 0 ? 64 : 128; }                         // output channels
constexpr int sr_dgrad_fwd_layer(int mode) { return mode == 0 ? 2 : mode == 1 ? 1 : 0; }    // k_sr_conv<LAYER> it inverts
constexpr size_t sr_dgrad_weight_bytes(int mode) { return (size_t)9 * sr_dgrad_cg(mode) * sr_dgrad_n(mode) * 4; }
constexpr int sr_wgrad_m(int mode) { return mode == 0 ? 64 : mode == 1 ? 256 : 128; }
constexpr int sr_wgrad_ci(int mode) { return mode == 0 ? 64 : 128; }
constexpr int sr_wgrad_slices(int mode) { return mode == 0 ? 64 : mode == 1 ? 16 : 32; }
constexpr int SR_SIMT_SLICES = 256;   // CTAs (= partials) of the SIMT reductions

// dgrad weight images of the three layers from the fp16 SW128 tiles of the packed model
cudaError_t launch_sr_pack_dgrad(const unsigned char *const tiles[3], unsigned char *const dst[3], cudaStream_t st);
cudaError_t launch_sr_dgrad(int mode, const SrDgradArgs &a, cudaStream_t st);
cudaError_t launch_sr_wgrad(int mode, const SrWgradArgs &a, cudaStream_t st);
// output stage at 2R: g [F,3,2R,2R] -> g_pre [F,2R,2R,64] = toRGB1 adjoint * y'(x1b); rgb_part (or nullptr) [slices][3*64+3]
cudaError_t launch_sr_bwd_out(const float *g, const __half *x1b, const float *rgb_w, const float *rgb_b, int F, int R2,
                              float *g_pre, float *rgb_part, cudaStream_t st);
// at R: g_img0 [F,R,R,3] = adjoint of the 2x up-sampled skip; g_r0 = g_img0 masked by toRGB0's clamp;
// rgb_part (or nullptr) [slices][3*128+3]
cudaError_t launch_sr_bwd_img0(const float *g, const __half *x0b, const float *rgb_w, const float *rgb_b, int F, int R,
                               float *g_img0, float *g_r0, float *rgb_part, cudaStream_t st);
// block0.conv0 (3 -> 128): grad_in [F,R,R,3] = adjoint of the conv on g_pre + g_img0; wgrad partials [slices][27*128]
cudaError_t launch_sr_in_dgrad(const float *g_pre, const float *w, const float *g_img0, int F, int R, float *grad_in, cudaStream_t st);
cudaError_t launch_sr_in_wgrad(const float *g_pre, const float *x, int F, int R, float *partial, cudaStream_t st);
// per-channel sums of g [F,P,C] and sum_p raw[p] sum_c g[p,c] (raw [P] shared or [F,P]; nullptr: 0) -> [slices][C+1]
cudaError_t launch_sr_chan_sums(const float *g, int C, int F, long long P, const float *raw, int raw_per_frame, float *partial,
                                cudaStream_t st);
// out[i] = sum_{s < S} part[s * stride + col0 + i] for i < n, s ascending
cudaError_t launch_sr_sum_cols(const float *part, int S, int stride, int col0, int n, float *out, cudaStream_t st);

}  // namespace gfpp
