// torso_sr_field.cuh -- tiling, shared-memory layout and helpers of the torso-SR field kernels: k_torso_sr (torso_sr_kernel.cu)
// and its point mode k_torso_sr_points (torso_sr_points_kernel.cu), which share their body (torso_sr_body.inc).
#pragma once
#include "torso_common.cuh"
#include "torso_sr_kernel.cuh"

namespace gfpp {
namespace tsr {

constexpr int TP = 128;    // pixels per tile
constexpr int NT = 256;
constexpr int KD0 = TORSO_SR_KD0, KC0 = TORSO_SR_KC0;
constexpr int LDT = 100;   // A-tile stride (>= 92, 16-byte aligned rows)
constexpr int LDE = 60;    // copy of the deform input (enc_x + head-aware encoding) for the canonical net
constexpr int NJAW = 14, NLM = NJAW + NJAW * 2 * 4;   // 126

struct Smem {
    float A[TP * LDT];
    float E[TP * LDE];
    float wd0[KD0 * 64], wd1[64 * 64], wc0[KC0 * 32], wc1[32 * 32];
    float wd2[2 * 64], wc2[4 * 32];
    float ha[TORSO_SR_HA_FLOATS];
    float x2[2 * TP];
    float alpha[TP], col[3 * TP], dxy[2 * TP];
    int mask[TP];
};

__device__ __forceinline__ float leaky002(float x) { return x > 0.f ? x : 0.02f * x; }


}  // namespace tsr
}  // namespace gfpp
