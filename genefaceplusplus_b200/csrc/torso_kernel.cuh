// torso_kernel.cuh -- argument block of the torso + composite epilogue (see torso_kernel.cu).
#pragma once
#include "common.cuh"

namespace gfpp {

struct TorsoArgs {
    int has_torso;
    GridMeta tor_gm;
    const float2 *tor_tab;
    // packed weights (device): k-major first/hidden layers, row-major narrow output layers
    const float *w_def0;   // [44][64]  (rows 42,43 zero)
    const float *w_def1;   // [64][64]
    const float *w_def2;   // [2][64]
    const float *w_can0;   // [76][32]  (rows 0-31 grid features, 32-73 enc_x, 74-75 zero)
    const float *w_can1;   // [32][32]
    const float *w_can2;   // [4][32]
    const float *bias_def; // [F][64] per-frame: pose + code columns of deform L0
    const float *bias_can; // [F][32] per-frame: pose + code columns of canonical L0
    const float *pose6;    // [F][6]
    const float *density_grid_torso;
    int grid_size;
    float density_thresh_torso, torso_shrink;
    const float *bg_coords; // [N,2]
    const float *bg_color;  // [N,3] or nullptr (=> 1)
    int n_frames, n_rays;
    const float *image;     // [F,N,3] premultiplied head colour
    const float *wsum;      // [F,N]
    float *rgb_map;         // [F,N,3] or nullptr
    unsigned char *rgb_u8;  // [F,N,3] (uint8)(int)(rgb*255) or nullptr
    float *alpha_map;       // [F,N] coverage A = ws + (1 - ws) * torso_alpha, or nullptr
    unsigned char *rgba_u8; // [F,N,4] 4-byte aligned: (uint8)(int)(P*255) x 3, (uint8)(int)(A*255); or nullptr
    float *torso_alpha;     // [F,N] or nullptr
    float *torso_rgb;       // [F,N,3] or nullptr
    float *deform;          // [F,N,2] or nullptr
    int *P_count;           // [F] or nullptr
    const unsigned char *w_tf32;  // TORSO_TF32_BYTES: tf32 hi / lo images of the four wide layers (below)
};

// tf32 hi / lo images of the four wide torso layers, read by k_epilogue's tensor cores: per layer hi then lo, each K/8 no-swizzle
// K8 blocks of N rows (tc.cuh, desc_tf32_k8).  K order (k_pack_tf32): deform L0 [enc_x 42 | 0 x 6]; canonical L0 [enc_x 42 |
// 0 x 6 | grid 32]; the grid block and both hidden layers permuted inside every 8 so that a k-step's A operand is an
// accumulator fragment as it stands (torso_kernel.cu).
struct TorsoTf32Layer { int N, K, hi; };
constexpr TorsoTf32Layer TORSO_TF32_D0 = {64, 48, 0}, TORSO_TF32_D1 = {64, 64, 2 * 64 * 48 * 4},
                         TORSO_TF32_C0 = {32, 80, TORSO_TF32_D1.hi + 2 * 64 * 64 * 4}, TORSO_TF32_C1 = {32, 32, TORSO_TF32_C0.hi + 2 * 32 * 80 * 4};
constexpr int TORSO_TF32_BYTES = TORSO_TF32_C1.hi + 2 * 32 * 32 * 4;   // 86 016
static_assert(TORSO_TF32_BYTES == 86016, "tf32 torso weight images");

size_t epilogue_smem_bytes();
cudaError_t launch_torso_frame_bias(const TorsoArgs &a, const float *w_def0, const float *w_can0, const float *code,
                                    int code_dim, float *bias_def, float *bias_can, cudaStream_t st);
cudaError_t launch_epilogue(const TorsoArgs &a, cudaStream_t st);
cudaError_t launch_pack_kmajor(const float *src, int ld, int row0, int col0, int N, int K, int Kpad, float *dst, cudaStream_t st);
cudaError_t launch_pack_tf32(const float *w_def0, int ld_def0, const float *w_def1, const float *w_can0, int ld_can0,
                             const float *w_can1, unsigned char *dst, cudaStream_t st);
cudaError_t launch_pack_rows(const float *src, int ld, int row0, int n_rows, int K, int dst_ld, float *dst, cudaStream_t st);
cudaError_t launch_fold_bias(const float *W, int ld, int col0, int nk, const float *v, int N, float *bias, cudaStream_t st);

}  // namespace gfpp
