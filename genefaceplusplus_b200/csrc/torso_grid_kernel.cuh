// torso_grid_kernel.cuh -- argument block of the torso field query (see torso_grid_kernel.cu).
#pragma once
#include "common.cuh"

namespace gfpp {

// Points come from `xy` [n,2] in [-1,1] or, when xy is null, from the cells of the H x H torso grid (n = H*H): point p is cell
// (x, y) = (p % H, p / H), the reference's tmp_grid_torso[y*H + x], placed exactly as radnerf_torso.py:221-227 does in fp32.
struct TorsoQueryArgs {
    GridMeta tor_gm;
    const float2 *tor_tab;
    // packed weights (device), the layouts of TorsoArgs (plain) / TorsoSrArgs (SR)
    const float *w_def0, *w_def1, *w_def2, *w_can0, *w_can1, *w_can2;
    const float *ha;        // SR only: head-aware encoder block (TORSO_SR_HA_FLOATS) or nullptr
    const float *bias_def;  // [64] the constant columns of deform L0 (frame-bias kernel with F = 1)
    const float *bias_can;  // [32] same through canonical L0
    float torso_shrink;
    uint32_t n;
    const float *xy;        // [n,2] or nullptr (cell mode)
    // cell mode
    uint32_t grid_size;     // H
    const float *noise;     // [H,H,2] in [0,1): meshgrid(x, y) order of the reference's rand_like draws
    float cell_scale, hgs;  // float(1 - 1/H), float(1/H)
    // outputs
    float *alpha;           // [n]
    float *color;           // [n,3] or nullptr
    float *deform;          // [n,2] or nullptr
};

cudaError_t launch_torso_query(const TorsoQueryArgs &q, cudaStream_t st);
cudaError_t launch_torso_sr_query(const TorsoQueryArgs &q, cudaStream_t st);

}  // namespace gfpp
