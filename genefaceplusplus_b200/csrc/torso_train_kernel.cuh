// torso_train_kernel.cuh -- the plain torso field's training forward and backward (gfpp.h section H), fp32 FFMA.
#pragma once
#include "common.cuh"

namespace gfpp {

constexpr int TORSO_TRAIN_TP = 128;     // points per tile (the tiling of k_torso_query)
constexpr int TORSO_TRAIN_CTAS = 132;   // persistent CTAs of the backward (fixed: the partial sums do not depend on the device)

// Re-laid-out weights and folded biases in the workspace (floats): the layouts gfpp_model_pack writes for the torso (TorsoArgs),
// then the two bias vectors k_torso_frame_bias writes for one frame.  k_torso_query reads them as it reads a packed model.
struct TorsoWt {
    static constexpr size_t wd0 = 0;                   // deform.0 enc_x columns, k-major   [44][64] (rows 42, 43 zero)
    static constexpr size_t wd1 = wd0 + 44 * 64;       // deform.1, k-major                 [64][64]
    static constexpr size_t wd2 = wd1 + 64 * 64;       // deform.2, rows                    [2][64]
    static constexpr size_t wc0 = wd2 + 2 * 64;        // canonical.0 [grid | enc_x], k-major [76][32] (rows 74, 75 zero)
    static constexpr size_t wc1 = wc0 + 76 * 32;       // canonical.1, k-major              [32][32]
    static constexpr size_t wc2 = wc1 + 32 * 32;       // canonical.2, rows                 [4][32]
    static constexpr size_t bias_def = wc2 + 4 * 32;   // [freq4(pose6) | code] . deform.0[:, 42:]^T     [64]
    static constexpr size_t bias_can = bias_def + 64;  // [freq4(pose6) | code] . canonical.0[:, 74:]^T  [32]
    static constexpr size_t total = bias_can + 32;
};

// Per-CTA partial sums of the backward (floats, one block per CTA).
struct TorsoPart {
    static constexpr size_t d0 = 0;                    // dW deform.0[:, 0:44]      [64][44] (columns 42, 43 unused)
    static constexpr size_t d1 = d0 + 64 * 44;         // dW deform.1               [64][64]
    static constexpr size_t d2 = d1 + 64 * 64;         // dW deform.2               [2][64]
    static constexpr size_t c0 = d2 + 2 * 64;          // dW canonical.0[:, 0:76]   [32][76] (columns 74, 75 unused)
    static constexpr size_t c1 = c0 + 32 * 76;         // dW canonical.1            [32][32]
    static constexpr size_t c2 = c1 + 32 * 32;         // dW canonical.2            [4][32]
    static constexpr size_t csd = c2 + 4 * 32;         // column sums of the deform.0 output gradient     [64]
    static constexpr size_t csc = csd + 64;            // column sums of the canonical.0 output gradient  [32]
    static constexpr size_t total = csc + 32;
};

struct TorsoTrainArgs {
    GridMeta gm;
    const float2 *tab;             // torso grid table [entries, 2]
    const float *w_def[3];         // [out, in] fp32: (64, din) (64, 64) (2, 64)
    const float *w_can[3];         // (32, 32 + din) (32, 32) (4, 32)
    const float *pose6;            // [6]
    const float *code;             // [code_dim] or nullptr
    int code_dim;                  // din = 42 + 54 + code_dim
    float shrink;
    uint32_t M;
    const float *xy;               // [M, 2]
    float *wt;                     // workspace: TorsoWt
    // backward
    const float *g_alpha, *g_color, *g_deform;   // [M], [M,3], [M,2]
    float *part;                   // TorsoPart::total * n_cta floats
    uint32_t n_cta;
    float2 *g_tab;
    float *g_def[3], *g_can[3], *g_code;
};

cudaError_t launch_torso_field_relayout(const TorsoTrainArgs &a, cudaStream_t st);
cudaError_t launch_torso_field_bwd(const TorsoTrainArgs &a, cudaStream_t st);
cudaError_t launch_torso_field_reduce(const TorsoTrainArgs &a, cudaStream_t st);

}  // namespace gfpp
