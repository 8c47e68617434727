// head_kernel.cuh -- argument block of the fused head renderer (see head_kernel.cu).
#pragma once
#include "common.cuh"

namespace gfpp {

constexpr int HEAD_TM = 128;      // samples per batch == ray slots per CTA
constexpr int HEAD_NT = 256;      // threads per CTA
constexpr int HEAD_NCHUNK = 11;
constexpr int HEAD_COARSE_WORDS = 1024;   // shared-memory slot for the coarse occupancy: 32 Ki bits = one cascade of 32^3   // weight chunks streamed per batch (see pack_head_weights in capi.cu)

struct HeadArgs {
    // ---- model ----
    GridMeta pos_gm, amb_gm;
    const float2 *pos_tab, *amb_tab;
    const float4 *pos_quads, *amb_quads;   // sector-packed corner layout (nullptr: use the reference layout)
    const uint4 *pos_octs, *amb_octs;      // fp16 oct layout (fp16 mode only; takes precedence over quads)
    const float *wide;              // concatenated k-major weight chunks, stream order
    int chunk_off[HEAD_NCHUNK];     // float offset of each chunk in `wide`
    int chunk_k[HEAD_NCHUNK];       // k-rows in each chunk (<= 72, multiple of 4)
    const float *narrow;            // [8][128]: ambient out rows 0-2, sigma row, color out rows 0-2, color-L0 bias
    MarchConst mc;
    const int *occ_bounds;          // device [6] tight occupied-cell bounds (or nullptr)
    const uint32_t *coarse_bits;    // device coarse occupancy (4x4x4 OR-pooled), cascade*(H/4)^3 bits, or nullptr
    int coarse_words;
    float aabb[6];
    float min_near, density_scale;
    int use_occ_box;                // 1: reject rays that miss the padded box of occupied voxels (cascade==1, aabb inside cube)
    // ---- frames ----
    int n_frames, n_rays;
    const float *rays_o, *rays_d;   // [F,N,3] or nullptr (then rays come from poses + intrinsics)
    const float *poses;             // [F,16]
    float fx, fy, cx, cy;
    int img_w;
    const float *cond_feat;         // [F,64]
    int max_steps;
    float T_thresh;
    // ---- outputs / state ----
    float *image;                   // [F,N,3] premultiplied head colour (before background)
    float *wsum;                    // [F,N]
    float *depth;                   // [F,N]
    float *rays_t;                  // [F,N] resume point of rays that outlive max_steps
    int *hist;                      // [F, max_steps+2] death-index histogram
    uint4 *hits;                    // [F*N][4] 64-byte records of the rays that reach a first sample, from k_ray_setup (HitRecord)
    int *n_hits;                    // [1]
    int *survivors;                 // [F*N] global ray ids still alive after max_steps samples
    int *n_survivors;               // [1]
    int *cursor;                    // [1] global work cursor
    int *B_total;                   // [F] per-frame sample cap produced by k_schedule
    int *valid_samples;             // [F] statistics (or nullptr)
    int pass;                       // 1 or 2
    unsigned long long *phase_cycles;  // optional [32]: per-phase cycle totals of thread 0 of every CTA (diagnostics)
    // ---- appended last so the offsets above stay put ----
    const float *noises;            // [F,N] in [0,1): jittered ray starts (k_ray_setup), or nullptr = start at near
    float *hit_ts;                  // [F*N][HIT_TS] pass-1 sample lists of the hit rays (k_march_list; read by k_head_v2), or nullptr
};

// k_march_list: per hit ray (indexed by ray id) the pre-step t of samples 2 .. HIT_TS (at most min(max_steps, HIT_TS) - 1 of them),
// then HIT_TS_END if the march ran off the ray before the list was full.  64 bytes per ray; the last word is never written
constexpr int HIT_TS = 16;
#define HIT_TS_END (-INFINITY)

// tensor-core variant: pre-swizzled 16-bit weight tiles (see pack_tc_weights in capi.cu)
constexpr int HEAD_TC_NCHUNK = 12;
// The weight stream of one batch: 12 tiles, always in this order (the kernel's schedule is compiled against this table,
// gfpp_model_pack fills the tiles from it).  rows x kc slice of layer `layer` starting at input column col0; k16 marks the
// no-swizzle K = 16 tile that pairs with the SH operand tile.
struct HeadTcChunk { int layer, rows, col0, kc, k16; };
constexpr HeadTcChunk kHeadTcChunks[HEAD_TC_NCHUNK] = {
    {0, 128, 0, 64, 0}, {0, 128, 64, 32, 0},     // ambient L0 (K = 96)
    {1, 128, 0, 64, 0}, {1, 128, 64, 64, 0},     // ambient L1
    {2, 128, 0, 64, 0},                          // sigma L0 (K = 64)
    {3, 128, 0, 64, 0}, {3, 128, 64, 64, 0},     // sigma L1
    {4, 144, 0, 64, 0}, {4, 144, 64, 64, 0},     // sigma L2: rows 0..127 geo, row 128 sigma, rest zero
    {5, 128, 16, 64, 0}, {5, 128, 80, 64, 0},    // color L0, geo columns 16..143
    {5, 128, 0, 16, 1}};                         // color L0, SH columns 0..15 (K16 tile)
constexpr int head_tc_chunk_bytes(int c) { return kHeadTcChunks[c].rows * (kHeadTcChunks[c].k16 ? 32 : 128); }
constexpr int head_tc_chunk_off(int c) { return c == 0 ? 0 : head_tc_chunk_off(c - 1) + head_tc_chunk_bytes(c - 1); }
constexpr int head_tc_chunk_ksteps(int c) { return kHeadTcChunks[c].k16 ? 1 : kHeadTcChunks[c].kc / 16; }
struct HeadTcArgs {
    const unsigned char *w_hi, *w_lo;       // the 12 streamed tiles back to back (head_tc_chunk_off), hi and lo images with identical layout
};
cudaError_t launch_head_tc(const HeadArgs &a, const HeadTcArgs &t, int precision, int total_hint, cudaStream_t st, bool train = false);
size_t head_tc_smem_bytes(bool split);

// ---- v2 (head_v2_kernel.cu): one CTA per SM, 2-3 row-owner slots of 128 samples sharing one weight stream ----
constexpr int V2_TILE_BYTES = 16384;            // one streamed weight tile: 128 rows x 64 k x 2 B (SW128)
// Streamed tiles of one super-batch, in order.  fp16: amb0 a (k 0-63: position features + conditioning 0-31), b (k 64-95: conditioning
// 32-63) | amb1 a,b | sig0 | sig1 a,b | fold a,b (W_fold = color L0 geo columns x sigma L2 geo rows, K = 128 over sigma L1's output);
// robust: every ambient tile is followed by its lo image.  Sigma L2 has no streamed tile: its sigma row is resident (V2_RES_SIGROW).
constexpr int V2_NTILE_X1 = 9, V2_NTILE_ROBUST = 13;
// Resident block (loaded once per CTA): the K16 SH tile of colour L0, then the narrow layers (K = 128, N <= 3, zero-padded to
// n = 8) as per-lane B-fragment images of mma.sync m16n8k16 (V2_NARROW_BYTES each, see k_pack_narrow_b): ambient out hi and lo,
// the sigma row of sigma L2, colour out
constexpr int V2_NARROW_BYTES = 2048;
constexpr int V2_RES_COLSH = 0, V2_RES_AMBN_HI = 4096, V2_RES_AMBN_LO = V2_RES_AMBN_HI + V2_NARROW_BYTES,
              V2_RES_SIGROW = V2_RES_AMBN_LO + V2_NARROW_BYTES, V2_RES_COLN = V2_RES_SIGROW + V2_NARROW_BYTES,
              V2_RES_BYTES = V2_RES_COLN + V2_NARROW_BYTES;
struct HeadV2Args {
    const unsigned char *w_stream;   // V2_NTILE_* tiles of V2_TILE_BYTES back to back
    const unsigned char *w_res;      // V2_RES_BYTES
    const unsigned char *cond_hi;    // [F,64] fp16: the frame's conditioning vector, pre-rounded (k_cond_images)
    const unsigned char *cond_lo;    // [F,64] fp16 residuals (robust mode)
    const float *pos_step;           // [16] per-level step of the 16-bit fixed-point position table (robust mode) or nullptr
};
cudaError_t launch_head_v2(const HeadArgs &a, const HeadV2Args &t, int precision, cudaStream_t st, bool train = false);
cudaError_t launch_cond_images(const float *cond_feat, int n_frames, void *cond_hi, void *cond_lo, cudaStream_t st);
size_t head_v2_smem_bytes(bool robust);

// ---- density query (k_density in head_kernel.cu): the head field up to the sigma net, no marching, no colour ----
// Points come from `xyzs` [n,3] or, when xyzs is null, from the occupancy cells in Morton order (n = C * H^3): point p is cell
// m = p % H^3 of cascade p / H^3, placed exactly as renderer.py:243-258 does on the CPU in fp32.
struct DensityArgs {
    uint32_t n;
    const float *xyzs;              // [n,3] or nullptr (cell mode)
    const float *cond;              // [64] one conditioning vector for every point
    float bound;                    // position grid bound (GridEncoder(..., bound=self.bound))
    // cell mode
    uint32_t grid_size;             // H
    const float *noise;             // [C,H,H,H,3] in [0,1): meshgrid(x,y,z) order of renderer.py:243 with S >= H
    float cell_scale[8], hgs[8];    // per cascade: float(bound_c - hgs_c) and float(hgs_c), hgs_c = bound_c / H
    // outputs
    float *sigma;                   // [n]: trunc_exp(h0) * out_scale
    float *geo;                     // [n,128] h[1:129], or nullptr (then the 128 geo columns are never computed)
    float out_scale;
};
// point p of a density query: xyzs[p], or the cell of Morton code p % H^3 in cascade p / H^3 placed exactly as renderer.py:246-258
// does in fp32 (xyzs = 2*c/(H-1) - 1; cas_xyzs = xyzs*(bound_c - hgs_c) + (noise*2 - 1)*hgs_c).  False (and zeros) past the end.
__device__ __forceinline__ bool density_point(const DensityArgs &d, uint32_t p, uint32_t H, uint32_t H3, float (&q)[3]) {
    q[0] = q[1] = q[2] = 0.f;
    if (p >= d.n) return false;
    if (d.xyzs) {
        q[0] = d.xyzs[3 * (size_t)p]; q[1] = d.xyzs[3 * (size_t)p + 1]; q[2] = d.xyzs[3 * (size_t)p + 2];
        return true;
    }
    const uint32_t cas = p / H3, m = p - cas * H3;
    const uint32_t c[3] = {compact3(m), compact3(m >> 1), compact3(m >> 2)};
    const float *nz = d.noise + ((((size_t)cas * H + c[0]) * H + c[1]) * H + c[2]) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float xs = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, (float)c[k]), (float)(H - 1)), 1.0f);
        const float r = __fmul_rn(__fsub_rn(__fmul_rn(nz[k], 2.0f), 1.0f), d.hgs[cas]);
        q[k] = __fadd_rn(__fmul_rn(xs, d.cell_scale[cas]), r);
    }
    return true;
}
// fp32 FFMA field (head_kernel.cu) / fp16 wgmma field over the fp16 operand images and oct tables (head_tc_kernel.cu)
cudaError_t launch_density(const HeadArgs &a, const DensityArgs &d, cudaStream_t st);
cudaError_t launch_density_tc(const HeadArgs &a, const HeadTcArgs &t, const DensityArgs &d, cudaStream_t st);

size_t head_smem_bytes();
// train: pass 1 with composite_rays_train's termination (k_head<true>, k_head_tc<.., .., true>, k_head_v2_train; gfpp_frozen_head)
cudaError_t launch_head(const HeadArgs &a, int total_hint, cudaStream_t st, bool train = false);
cudaError_t launch_ray_setup(const HeadArgs &a, cudaStream_t st);
cudaError_t launch_march_list(const HeadArgs &a, cudaStream_t st);
cudaError_t launch_dump_rays(const HeadArgs &a, float *rays_o, float *rays_d, cudaStream_t st);
cudaError_t launch_schedule(const int *hist, int n_frames, int n_rays, int max_steps, int *B_total, cudaStream_t st);

}  // namespace gfpp
