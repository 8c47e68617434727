// field_train_kernel.cuh -- the head field's training forward and backward (gfpp.h section G), fp32 FFMA.
#pragma once
#include "common.cuh"

namespace gfpp {

constexpr int FIELD_TP = 64;          // points per tile
constexpr int FIELD_CTAS = 132;       // persistent CTAs of the backward (fixed: the partial sums do not depend on the device)

// Re-laid-out weights in the workspace (floats): k-major transposes of the wide layers' forward operands, then the folded biases.
struct FieldWt {
    static constexpr size_t a0 = 0;                  // ambient_net.0 pos columns 0..31     [32][128]
    static constexpr size_t a1 = a0 + 32 * 128;      // ambient_net.1                       [128][128]
    static constexpr size_t s0 = a1 + 128 * 128;     // sigma_net.0                         [64][128]
    static constexpr size_t s1 = s0 + 64 * 128;      // sigma_net.1                         [128][128]
    static constexpr size_t s2 = s1 + 128 * 128;     // sigma_net.2 geo rows 1..128         [128][128]
    static constexpr size_t c0 = s2 + 128 * 128;     // color_net.0 columns 0..143          [144][128]
    static constexpr size_t bias_a0 = c0 + 144 * 128;  // cond . ambient_net.0[:, 32:96]^T  [128]
    static constexpr size_t bias_c0 = bias_a0 + 128;   // code . color_net.0[:, 144:]^T     [128]
    static constexpr size_t total = bias_c0 + 128;
};

// Per-CTA partial sums of the backward (floats, one block per CTA).
struct FieldPart {
    static constexpr size_t a0 = 0;                  // dW ambient_net.0[:, 0:32]   [128][32]
    static constexpr size_t a1 = a0 + 128 * 32;      // dW ambient_net.1            [128][128]
    static constexpr size_t a2 = a1 + 128 * 128;     // dW ambient_net.2            [3][128]
    static constexpr size_t s0 = a2 + 3 * 128;       // dW sigma_net.0              [128][64]
    static constexpr size_t s1 = s0 + 128 * 64;      // dW sigma_net.1              [128][128]
    static constexpr size_t s2 = s1 + 128 * 128;     // dW sigma_net.2              [129][128]
    static constexpr size_t c0 = s2 + 129 * 128;     // dW color_net.0[:, 0:144]    [128][144]
    static constexpr size_t c1 = c0 + 128 * 144;     // dW color_net.1              [3][128]
    static constexpr size_t csa = c1 + 3 * 128;      // column sums of the ambient_net.0 output gradient  [128]
    static constexpr size_t csc = csa + 128;         // column sums of the color_net.0 output gradient    [128]
    static constexpr size_t total = csc + 128;
};

struct FieldArgs {
    GridMeta pos_gm, amb_gm;
    const float2 *pos_tab, *amb_tab;
    const float *w[8];             // [out, in] fp32: ambient 0..2, sigma 3..5, colour 6..7
    const float *cond;             // [64]
    const float *code;             // [ind_dim] or nullptr
    int ind_dim, amb_dim;
    float bound;
    uint32_t M;
    const float *xyzs, *dirs;      // [M,3]
    float *wt;                     // workspace: FieldWt
    // forward outputs (k_field_fwd)
    float *sigma, *color, *ambient;
    // backward (k_field_bwd, k_field_reduce)
    const float *g_sigma, *g_color, *g_ambient;
    float *part;                   // FieldPart::total * n_cta floats
    uint32_t n_cta;
    float2 *g_pos_tab, *g_amb_tab;
    float *g_w[8];
    float *g_cond, *g_code;
};

cudaError_t launch_field_relayout(const FieldArgs &a, cudaStream_t st);
cudaError_t launch_field_fwd(const FieldArgs &a, cudaStream_t st);
cudaError_t launch_field_bwd(const FieldArgs &a, cudaStream_t st);
cudaError_t launch_field_reduce(const FieldArgs &a, cudaStream_t st);

}  // namespace gfpp
