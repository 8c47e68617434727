// grid_half.cuh -- launch interface of the half-table grid encoder (grid_half_kernels.cu, gfpp.h section (L)).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace gfpp {

// What the reference kernels take as arguments (gridencoder.cu:88-98): the level offsets and the raw S / H, from which every
// level constant is derived on the device.  Passed by value.
struct HalfGridArgs {
    uint32_t offset[GFPP_MAX_LEVELS + 1];   // table offsets in entries (half2 slots)
    uint32_t L;
    float S;
    uint32_t H;
    uint32_t gridtype;                      // 0 hash, 1 tiled
    uint32_t align_corners;
    uint32_t interp;                        // 0 linear, 1 smoothstep
};

cudaError_t launch_grid_half_forward(const HalfGridArgs &g, uint32_t D, const float *inputs, const void *table, void *outputs, void *dy_dx,
                                     uint32_t B, cudaStream_t st);
cudaError_t launch_grid_half_backward(const HalfGridArgs &g, uint32_t D, const void *grad, const float *inputs, void *grad_table,
                                      const void *dy_dx, void *grad_inputs, uint32_t B, int *launches, cudaStream_t st);

}  // namespace gfpp
