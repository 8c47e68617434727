// ops.cuh -- host launchers of the kernels outside the fused renderer and the training fields: the per-op mirror of the reference
// extensions, the training-side ops, the occupancy-grid refresh, the torso pass, the I420 conversion and the tensor-core weight
// packing.  Each defining file includes this header, so a declaration that drifts from its definition does not compile.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace gfpp {

// ---- ops_kernels.cu ----
cudaError_t launch_near_far(const float *rays_o, const float *rays_d, const float *aabb, uint32_t N, float min_near, float *nears,
                            float *fars, cudaStream_t st);
cudaError_t launch_march_rays(const MarchConst &mc, uint32_t n_alive, uint32_t n_step, const int32_t *rays_alive, const float *rays_t,
                              const float *rays_o, const float *rays_d, const float *fars, float *xyzs, float *dirs, float *deltas,
                              const float *noises, cudaStream_t st);
cudaError_t launch_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t *rays_alive, float *rays_t, const float *sigmas,
                                  const float *rgbs, const float *deltas, float *weights_sum, float *depth, float *image, cudaStream_t st);
cudaError_t launch_grid_encode(const GridMeta &gm, const float *inputs, const float *table, float *outputs, uint32_t B, cudaStream_t st);
cudaError_t launch_sh_encode(const float *inputs, float *outputs, uint32_t B, uint32_t degree, cudaStream_t st);
cudaError_t launch_freq_encode(const float *inputs, uint32_t B, uint32_t D, uint32_t C, float *outputs, cudaStream_t st);
cudaError_t launch_occupancy_bounds(const uint8_t *bits, uint32_t n_bytes, uint32_t H3, int *bounds, cudaStream_t st);
cudaError_t launch_coarse_occupancy(const uint8_t *bits, uint32_t C, uint32_t H, uint32_t *coarse, cudaStream_t st);
cudaError_t launch_pack_quads(const GridMeta &gm, const float *table, float *quads, uint32_t total, cudaStream_t st);
cudaError_t launch_pack_octs(const GridMeta &gm, const float *table, void *octs, uint32_t total, cudaStream_t st);
cudaError_t launch_pack_octs_i16(const GridMeta &gm, const float *table, void *octs, uint32_t total, uint32_t *scratch, float *step,
                                 cudaStream_t st);

// ---- tc_pack.cu ----
cudaError_t launch_pack_tc_tile(const float *W, int ld, int row0, int col0, int N, int kc, int dst_row0, int k16, int bf16,
                                unsigned char *hi, unsigned char *lo, cudaStream_t st);
cudaError_t launch_pack_fold_tile(const float *Wc, int ldc, int c0, const float *Ws, unsigned char *tiles, int tile_bytes, cudaStream_t st);
cudaError_t launch_pack_narrow_b(const float *W, int ld, int N, unsigned char *hi, unsigned char *lo, cudaStream_t st);
cudaError_t launch_tc_selftest(const float *A, int K, const unsigned char *wt_hi, const unsigned char *wt_lo, int N, int nt64,
                               int k16_tail, int precision, float *out, cudaStream_t st);

// ---- train_kernels.cu ----
size_t march_train_scratch_bytes(uint32_t N);
cudaError_t launch_march_rays_train(const MarchConst &mc, const float *rays_o, const float *rays_d, const float *nears, const float *fars,
                                    const float *noises, uint32_t N, uint32_t M, uint32_t max_steps, float *xyzs, float *dirs, float *deltas,
                                    int *rays, int *counter, int *scratch, int *n_launches, cudaStream_t st);
cudaError_t launch_march_rays_train_backward(const float *grad_xyzs, const float *grad_dirs, const int *rays, const float *deltas, uint32_t N,
                                             uint32_t M, float *grad_rays_o, float *grad_rays_d, cudaStream_t st);
cudaError_t launch_composite_train_forward(const float *sigmas, const float *rgbs, const float *ambient, const float *deltas, const int *rays,
                                           uint32_t M, uint32_t N, float T_thresh, float *weights_sum, float *ambient_sum, float *depth,
                                           float *image, cudaStream_t st);
cudaError_t launch_composite_train_backward(const float *grad_weights_sum, const float *grad_ambient_sum, const float *grad_image,
                                            const float *sigmas, const float *rgbs, const float *ambient, const float *deltas, const int *rays,
                                            const float *weights_sum, const float *ambient_sum, const float *image, uint32_t M, uint32_t N,
                                            float T_thresh, float *grad_sigmas, float *grad_rgbs, float *grad_ambient, cudaStream_t st);
cudaError_t launch_grid_encode_dydx(const GridMeta &gm, const float *inputs, const float *table, float *outputs, float *dy_dx, uint32_t B,
                                    cudaStream_t st);
cudaError_t launch_grid_backward(const GridMeta &gm, const float *grad, const float *inputs, float *grad_table, const float *dy_dx,
                                 float *grad_inputs, uint32_t B, int *n_launches, cudaStream_t st);
cudaError_t launch_grad_tv(const GridMeta &gm, const float *inputs, const float *table, float *grad_table, float weight, uint32_t B,
                           cudaStream_t st);
cudaError_t launch_packbits(const float *grid, uint32_t N, float thresh, uint8_t *bitfield, cudaStream_t st);
cudaError_t launch_morton3D(const int *coords, uint32_t N, int *indices, cudaStream_t st);
cudaError_t launch_morton3D_invert(const int *indices, uint32_t N, int *coords, cudaStream_t st);
cudaError_t launch_morton3D_dilation(const float *grid, uint32_t C, uint32_t H, float *out, cudaStream_t st);
cudaError_t launch_sph_from_ray(const float *rays_o, const float *rays_d, float radius, uint32_t N, float *coords, cudaStream_t st);

// ---- grid_kernels.cu ----
uint32_t dilate_ema_blocks(uint32_t C, uint32_t H);
cudaError_t launch_grid_refresh_tail(const float *tmp, uint32_t C, uint32_t H, float decay, float density_thresh, float *grid,
                                     double *partial, float *mean_out, float *thresh_dev, uint8_t *bitfield, int *n_launches, cudaStream_t st);
uint32_t torso_dilate_ema_blocks(uint32_t H);
cudaError_t launch_torso_grid_tail(const float *tmp, uint32_t H, float decay, float density_thresh, float *grid, double *partial,
                                   float *mean_out, float *thresh_dev, int *n_launches, cudaStream_t st);
cudaError_t launch_mark_untrained(const float *poses, uint32_t B, float rx, float ry, const float *cell_scale, const float *pad, uint32_t C,
                                  uint32_t H, float *grid, cudaStream_t st);

// ---- torso_pass_kernels.cu ----
uint32_t torso_mask_tiles(uint32_t N);
cudaError_t launch_torso_mask(const float *grid, uint32_t G, float thr, const float *xy, const float *image, const float *wsum, uint32_t N,
                              int32_t *idx, int32_t *slot, float *xy_m, float *image_m, float *wsum_m, int32_t *count, int *tile_sums,
                              cudaStream_t st);
cudaError_t launch_torso_composite_fwd(const int32_t *slot, uint32_t N, const float *alpha, const float *color, const float *image,
                                       const float *wsum, const float *bg, uint32_t bg_mode, float *torso_alpha_map, float *torso_rgb_map,
                                       float *rgb_map, cudaStream_t st);
cudaError_t launch_torso_composite_bwd(const int32_t *idx, uint32_t M, const float *alpha, const float *color, const float *image,
                                       const float *wsum, const float *bg, uint32_t bg_mode, const float *g_ta, const float *g_trgb,
                                       const float *g_rgb, float *grad_alpha, float *grad_color, cudaStream_t st);

// ---- video_kernels.cu ----
cudaError_t launch_rgb_u8_to_i420(const uint8_t *rgb, uint32_t F, uint32_t H, uint32_t W, uint8_t *out, cudaStream_t st);

}  // namespace gfpp
