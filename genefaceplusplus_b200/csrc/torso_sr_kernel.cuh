// torso_sr_kernel.cuh -- argument block of the torso-SR field + composite (see torso_sr_kernel.cu).
#pragma once
#include "common.cuh"

namespace gfpp {

struct TorsoSrArgs {
    GridMeta tor_gm;
    const float2 *tor_tab;
    // packed weights (device): k-major first/hidden layers, row-major narrow output layers
    const float *w_def0;   // [60][64]  rows 0-41 enc_x, 42-57 head-aware encoding (zero rows without it), 58-59 zero
    const float *w_def1;   // [64][64]
    const float *w_def2;   // [2][64]
    const float *w_can0;   // [92][32]  rows 0-31 grid features, 32-73 enc_x, 74-89 head-aware encoding, 90-91 zero
    const float *w_can1;   // [32][32]
    const float *w_can2;   // [4][32]
    const float *ha;       // head-aware encoder 4 -> 16 -> 32 -> 16, k-major + biases (TORSO_SR_HA_FLOATS), or nullptr
    const float *bias_def; // [F][64] per-frame: torso code + freq-encoded jaw landmarks through deform L0
    const float *bias_can; // [F][32] same through canonical L0
    const float *density_grid_torso;
    int grid_size;
    float density_thresh_torso, torso_shrink;
    const float *bg_coords; // [N,2]
    const float *bg_color;  // [N,3] or nullptr (=> 1)
    int n_frames, n_rays;
    const float *image;     // [F,N,3] premultiplied head colour
    const float *wsum;      // [F,N]
    float *rgb_map;         // [F,N,3]
    float *torso_alpha;     // [F,N] or nullptr
    float *torso_rgb;       // [F,N,3] or nullptr
    float *deform;          // [F,N,2] or nullptr
    int *P_count;           // [F] or nullptr (must be zeroed by the caller)
};

// layout of the head-aware encoder block: W0 [4][16] | b0 [16] | W1 [16][32] | b1 [32] | W2 [32][16] | b2 [16]
constexpr int TORSO_SR_HA_W0 = 0, TORSO_SR_HA_B0 = 64, TORSO_SR_HA_W1 = 80, TORSO_SR_HA_B1 = 592, TORSO_SR_HA_W2 = 624,
              TORSO_SR_HA_B2 = 1136, TORSO_SR_HA_FLOATS = 1152;
constexpr int TORSO_SR_KD0 = 60, TORSO_SR_KC0 = 92;

cudaError_t launch_torso_sr_frame_bias(const float *lm68, int n_frames, const float *w_def0, const float *w_can0, const float *code,
                                       int code_dim, int head_aware, float *bias_def, float *bias_can, cudaStream_t st);
cudaError_t launch_torso_sr(const TorsoSrArgs &a, cudaStream_t st);
// k_torso_sr's field at explicit points (n_frames 1, bg_coords = the points, no mask, image / wsum per point or both nullptr):
// writes torso_alpha [n], torso_rgb [n,3] (the field's colour) and deform [n,2]; no composite.
cudaError_t launch_torso_sr_points(const TorsoSrArgs &a, cudaStream_t st);

}  // namespace gfpp
