// torso_sr_points_kernel.cu -- k_torso_sr_points: the torso-SR render epilogue's field (k_torso_sr) in its point mode, the forward of
// the trainable torso-SR field (gfpp.h section I).  It is k_torso_sr's own body (torso_sr_body.inc) with POINTS = true, kept in its
// own translation unit so that k_torso_sr is compiled alone, exactly as before the point mode existed.
#include "launch.cuh"
#include "torso_sr_field.cuh"
#include "torso_sr_kernel.cuh"

namespace gfpp {

using namespace torsoc;
using namespace tsr;

__global__ void __launch_bounds__(256, 1) k_torso_sr_points(const __grid_constant__ TorsoSrArgs a) {
    constexpr bool POINTS = true;
#include "torso_sr_body.inc"
}

cudaError_t launch_torso_sr_points(const TorsoSrArgs &a, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(k_torso_sr_points, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem));
    if (e != cudaSuccess) return e;
    const int tiles = (a.n_rays + TP - 1) / TP;
    int blocks = sm_count();
    if (tiles < blocks) blocks = tiles > 0 ? tiles : 1;
    k_torso_sr_points<<<blocks, NT, sizeof(Smem), st>>>(a);
    return cudaGetLastError();
}

}  // namespace gfpp
