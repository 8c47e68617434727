// field_train_tc_kernel.cuh -- the head field's training forward and backward on fp16 wgmma with fp32 accumulation (gfpp.h section J).
#pragma once
#include "field_train_kernel.cuh"

namespace gfpp {

constexpr int FIELD_TC_TP = 128;      // points per tile: two M = 64 halves, one per warpgroup

// fp16 weight images in the workspace (bytes): SW128 K-major operand tiles of [rows x 64 elements] (tc.cuh), K-tile t of an image
// `rows * 128` bytes after tile 0.  The forward images have rows = outputs and K = inputs; the *T images are the operands of the
// input-gradient product dX = dY W: rows = inputs, K = outputs.  Rows / columns past the layer's are zero.
struct FieldTcImg {
    static constexpr uint32_t T = 16384;             // one [128 x 64] tile
    static constexpr uint32_t a0 = 0;                // ambient_net.0[:, 0:32]               1 tile
    static constexpr uint32_t a1 = a0 + T;           // ambient_net.1                        2 tiles
    static constexpr uint32_t s0 = a1 + 2 * T;       // sigma_net.0                          1 tile
    static constexpr uint32_t s1 = s0 + T;           // sigma_net.1                          2 tiles
    static constexpr uint32_t s2 = s1 + 2 * T;       // sigma_net.2 geo rows 1..128          2 tiles
    static constexpr uint32_t c0 = s2 + 2 * T;       // color_net.0: geo columns 16..143 (2 tiles), then SH columns 0..15 (1 tile)
    static constexpr uint32_t c0T = c0 + 3 * T;      // color_net.0[:, 16:144]^T             2 tiles
    static constexpr uint32_t s2T = c0T + 2 * T;     // sigma_net.2[1:129]^T                 2 tiles
    static constexpr uint32_t s1T = s2T + 2 * T;     // sigma_net.1^T                        2 tiles
    static constexpr uint32_t s0T = s1T + 2 * T;     // sigma_net.0^T         [64 rows]      2 tiles of 8 KB
    static constexpr uint32_t a1T = s0T + T;         // ambient_net.1^T                      2 tiles
    static constexpr uint32_t a0T = a1T + 2 * T;     // ambient_net.0[:, 0:32]^T [64 rows, 32 used]  2 tiles of 8 KB
    static constexpr uint32_t bias = a0T + T;        // fp32: cond . ambient_net.0[:, 32:96]^T [128], code . color_net.0[:, 144:]^T [128]
    static constexpr uint32_t total = bias + 256 * 4;
};

// FieldArgs as section G fills it, with f.wt -> the two folded biases and f.part / f.n_cta -> FieldPart blocks (k_field_reduce reads
// them unchanged), plus the weight images.
struct FieldTcArgs {
    FieldArgs f;
    unsigned char *img;            // workspace: FieldTcImg
};

cudaError_t launch_field_tc_relayout(const FieldTcArgs &a, cudaStream_t st);
cudaError_t launch_field_tc_fwd(const FieldTcArgs &a, cudaStream_t st);
cudaError_t launch_field_tc_bwd(const FieldTcArgs &a, cudaStream_t st);

}  // namespace gfpp
