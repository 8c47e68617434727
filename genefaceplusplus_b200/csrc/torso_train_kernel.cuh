// torso_train_kernel.cuh -- the training forward and backward of both torso fields, fp32 FFMA: the plain torso's (gfpp.h section H,
// SR = false) and the torso-SR model's (section I, SR = true).
#pragma once
#include "common.cuh"
#include "torso_sr_kernel.cuh"

namespace gfpp {

constexpr int TORSO_TRAIN_TP = 128;     // points per tile (the tiling of k_torso_query and k_torso_sr)
constexpr int TORSO_TRAIN_CTAS = 132;   // persistent CTAs of the backward (fixed: the partial sums do not depend on the device)

template <bool SR> struct TorsoShape;
// plain: deform input [enc_x 42 | pad 2], canonical input [grid 32 | enc_x 42 | pad 2]
template <> struct TorsoShape<false> { static constexpr int KD0 = 44, KC0 = 76, LDC = 84; };
// SR: deform input [enc_x 42 | head-aware 16 | pad 2], canonical input [grid 32 | the same]
template <> struct TorsoShape<true> { static constexpr int KD0 = TORSO_SR_KD0, KC0 = TORSO_SR_KC0, LDC = 100; };

// Re-laid-out weights and folded biases in the workspace (floats): the layouts gfpp_model_pack (TorsoArgs) or gfpp_torso_sr_pack
// (TorsoSrArgs) writes, then the two bias vectors k_torso_frame_bias or k_torso_sr_frame_bias writes for one frame.  The forward
// (k_torso_query, or k_torso_sr's point mode) reads them as it reads a packed model.
template <bool SR> struct TorsoWt {
    static constexpr size_t wd0 = 0;                                  // deform.0 columns of the deform input, k-major  [KD0][64]
    static constexpr size_t wd1 = wd0 + TorsoShape<SR>::KD0 * 64;     // deform.1, k-major                              [64][64]
    static constexpr size_t wd2 = wd1 + 64 * 64;                      // deform.2, rows                                 [2][64]
    static constexpr size_t wc0 = wd2 + 2 * 64;                       // canonical.0 [grid | deform input], k-major     [KC0][32]
    static constexpr size_t wc1 = wc0 + TorsoShape<SR>::KC0 * 32;     // canonical.1, k-major                           [32][32]
    static constexpr size_t wc2 = wc1 + 32 * 32;                      // canonical.2, rows                              [4][32]
    static constexpr size_t ha = wc2 + 4 * 32;                        // SR: head-aware encoder (TORSO_SR_HA_* layout)  [1152]
    static constexpr size_t bias_def = ha + (SR ? TORSO_SR_HA_FLOATS : 0);   // constant columns . deform.0[:, 42:]^T    [64]
    static constexpr size_t bias_can = bias_def + 64;                 // constant columns . canonical.0[:, 74:]^T       [32]
    static constexpr size_t total = bias_can + 32;
};

// Per-CTA partial sums of the backward (floats, one block per CTA); [out][in] layouts.
template <bool SR> struct TorsoPart {
    static constexpr size_t d0 = 0;                                   // dW deform.0 at the deform-input columns  [64][KD0]
    static constexpr size_t d1 = d0 + 64 * TorsoShape<SR>::KD0;       // dW deform.1               [64][64]
    static constexpr size_t d2 = d1 + 64 * 64;                        // dW deform.2               [2][64]
    static constexpr size_t c0 = d2 + 2 * 64;                         // dW canonical.0 at the [grid | deform input] columns  [32][KC0]
    static constexpr size_t c1 = c0 + 32 * TorsoShape<SR>::KC0;       // dW canonical.1            [32][32]
    static constexpr size_t c2 = c1 + 32 * 32;                        // dW canonical.2            [4][32]
    static constexpr size_t csd = c2 + 4 * 32;                        // column sums of the deform.0 output gradient     [64]
    static constexpr size_t csc = csd + 64;                           // column sums of the canonical.0 output gradient  [32]
    static constexpr size_t hw0 = csc + 32;                           // SR: dW head-aware.0 [16][4]
    static constexpr size_t hb0 = hw0 + 16 * 4;                       //     db head-aware.0 [16]
    static constexpr size_t hw1 = hb0 + 16;                           //     dW head-aware.2 [32][16]
    static constexpr size_t hb1 = hw1 + 32 * 16;                      //     db head-aware.2 [32]
    static constexpr size_t hw2 = hb1 + 32;                           //     dW head-aware.4 [16][32]
    static constexpr size_t hb2 = hw2 + 16 * 32;                      //     db head-aware.4 [16]
    static constexpr size_t total = SR ? hb2 + 16 : hw0;
};

struct TorsoTrainArgs {
    GridMeta gm;
    const float2 *tab;             // torso grid table [entries, 2]
    const float *w_def[3];         // [out, in] fp32: (64, din) (64, 64) (2, 64)
    const float *w_can[3];         // (32, 32 + din) (32, 32) (4, 32)
    const float *cond;             // plain: pose6 [6]; SR: lm68 [136]
    const float *code;             // [code_dim] or nullptr
    int code_dim;                  // din = 42 + 54 + code_dim (plain), 42 + code_dim + 126 (+ 16 with head_aware) (SR)
    float shrink;
    uint32_t M;
    const float *xy;               // [M, 2]
    float *wt;                     // workspace: TorsoWt<SR>
    // backward
    const float *g_alpha, *g_color, *g_deform;   // [M], [M,3], [M,2]
    float *part;                   // TorsoPart<SR>::total * n_cta floats
    uint32_t n_cta;
    float2 *g_tab;
    float *g_def[3], *g_can[3], *g_code;
    // SR only: zero and null for the plain field
    int head_aware;
    const float *ha_w[3], *ha_b[3];   // head_color_weights_encoder (16,4) (32,16) (16,32) and biases; nullptr without head_aware
    const float *image, *wsum;     // [M, 3], [M] or both nullptr (the encoder then sees zeros)
    float *g_ha_w[3], *g_ha_b[3];
};

// SR = false launches k_torso_field_*, SR = true k_torso_sr_field_*
template <bool SR> cudaError_t launch_torso_field_relayout(const TorsoTrainArgs &a, cudaStream_t st);
template <bool SR> cudaError_t launch_torso_field_bwd(const TorsoTrainArgs &a, cudaStream_t st);
template <bool SR> cudaError_t launch_torso_field_reduce(const TorsoTrainArgs &a, cudaStream_t st);

}  // namespace gfpp
