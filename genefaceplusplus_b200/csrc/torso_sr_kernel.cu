// torso_sr_kernel.cu -- torso field + final composite of the torso-SR checkpoints (`lm3d_radnerf_torso_sr.yaml`).
//
// Replaces RADNeRFTorsowithSR.forward_torso and the composite of its render() (modules/radnerfs/radnerf_torso_sr.py:75-113,
// 196-228).  Against the plain torso model (torso_kernel.cu) the field is conditioned on the freq-encoded JAW landmarks
// (lm68 points 5..11, 14 -> 126 values) instead of the head pose, and -- `torso_head_aware` -- on a per-pixel 4 -> 16 -> 32 ->
// 16 encoding (LeakyReLU 0.02, with biases) of the rendered head colour and alpha at that pixel:
//     h = [freq10(0.8 x) 42 | code 8 | freq4(jaw) 126 | head-aware 16]   ->  deform 64-64-2,  x' = clamp(x + dx)
//     [tiled2D(x') 32 | h]                                               ->  canonical 32-32-4 -> sigmoid alpha, rgb
// Per-frame constants (code, landmarks) are folded into per-frame bias vectors (k_torso_sr_frame_bias); the per-pixel GEMMs see
// 58 (deform) / 90 (canonical) columns.  Same tiling as k_epilogue: persistent, 128-pixel tiles, tiles without torso pixels
// skip the MLPs; fp32 FFMA tile GEMMs out of shared memory; accurate sinf; grid_sample restated.
#include "launch.cuh"
#include "torso_common.cuh"
#include "torso_sr_field.cuh"
#include "torso_sr_kernel.cuh"

namespace gfpp {

using namespace torsoc;
using namespace tsr;

// per-frame bias vectors: columns [code | freq4(jaw landmarks)] of the first deform / canonical layers
__global__ void k_torso_sr_frame_bias(const float *__restrict__ lm68 /*[F,136]*/, const float *__restrict__ w_def0 /*[64,din]*/,
                                      const float *__restrict__ w_can0 /*[32,32+din]*/, const float *__restrict__ code, int code_dim,
                                      int head_aware, float *__restrict__ bias_def, float *__restrict__ bias_can) {
    const int f = blockIdx.x, j = threadIdx.x;
    __shared__ float h[160];
    const int nh = code_dim + NLM;
    if (j < code_dim) h[j] = code ? code[j] : 0.f;
    else if (j < nh) h[j] = freq_entry(lm68 + (size_t)f * 136 + 10, NJAW, j - code_dim);   // points 5..11 of [68,2]
    __syncthreads();
    const int din = 42 + nh + (head_aware ? 16 : 0);
    if (j < 64) {
        float s = 0.f;
        for (int k = 0; k < nh; ++k) s = fmaf(w_def0[j * din + 42 + k], h[k], s);
        bias_def[(size_t)f * 64 + j] = s;
    }
    if (j < 32) {
        float s = 0.f;
        for (int k = 0; k < nh; ++k) s = fmaf(w_can0[j * (32 + din) + 32 + 42 + k], h[k], s);
        bias_can[(size_t)f * 32 + j] = s;
    }
}

__global__ void __launch_bounds__(256, 1) k_torso_sr(const __grid_constant__ TorsoSrArgs a) {
    constexpr bool POINTS = false;
#include "torso_sr_body.inc"
}

cudaError_t launch_torso_sr_frame_bias(const float *lm68, int n_frames, const float *w_def0, const float *w_can0, const float *code,
                                       int code_dim, int head_aware, float *bias_def, float *bias_can, cudaStream_t st) {
    if (code_dim < 0 || code_dim + NLM > 160) return cudaErrorInvalidValue;
    k_torso_sr_frame_bias<<<n_frames, 160, 0, st>>>(lm68, w_def0, w_can0, code, code_dim, head_aware, bias_def, bias_can);
    return cudaGetLastError();
}

cudaError_t launch_torso_sr(const TorsoSrArgs &a, cudaStream_t st) {
    static_assert(sizeof(Smem) <= 227 * 1024, "torso-SR epilogue exceeds the per-CTA shared memory limit");
    // function attributes are per device: set on every launch, never cached process-wide
    cudaError_t e = cudaFuncSetAttribute(k_torso_sr, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    const int tiles = a.n_frames * ((a.n_rays + TP - 1) / TP);
    int blocks = sm_count();
    if (tiles < blocks) blocks = tiles > 0 ? tiles : 1;
    k_torso_sr<<<blocks, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

}  // namespace gfpp
