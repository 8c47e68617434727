// grid_kernels.cu -- occupancy-grid maintenance behind gfpp.h section (E): the device half of NeRFRenderer.update_extra_state
// (modules/radnerfs/renderer.py:201-278) after the density query (k_density, head_kernel.cu), and mark_untrained_grid
// (renderer.py:131-199), and the torso grid's dilation + EMA + mean after the torso query (k_torso_query / k_torso_sr_query,
// torso_grid_kernel.cu).  Everything is stream-ordered and deterministic: fixed work per block, fixed reduction trees, no atomics.
#include "common.cuh"
#include "launch.cuh"

namespace gfpp {

namespace {

constexpr int RED_NT = 256;
constexpr int RED_PER_THREAD = 16;
constexpr int RED_CELLS = RED_NT * RED_PER_THREAD;   // cells per block of k_dilate_ema

// sum of `v` over the block in a fixed order (warp butterfly, then warp 0 over the warp sums); valid in thread 0
__device__ __forceinline__ double block_sum(double v, double *sh) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) sh[wid] = v;
    __syncthreads();
    v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    if (wid == 0)
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// renderer.py:266-272: tmp = morton3D_dilation(tmp) (max over the cell and its 6 neighbours); where grid >= 0 and tmp >= 0:
// grid = max(grid * decay, tmp); then this block's share of sum(clamp(grid, 0)) in double.
__global__ void __launch_bounds__(RED_NT) k_dilate_ema(const float *__restrict__ tmp, uint32_t C, uint32_t H, float decay,
                                                       float *__restrict__ grid, double *__restrict__ partial) {
    __shared__ double sh[RED_NT / 32];
    const uint32_t H3 = H * H * H, total = C * H3;
    double acc = 0.0;
    const uint32_t base = blockIdx.x * RED_CELLS;
#pragma unroll 4
    for (int k = 0; k < RED_PER_THREAD; ++k) {
        const uint32_t n = base + k * RED_NT + threadIdx.x;
        if (n >= total) break;
        const uint32_t c = n / H3, ind = n - c * H3;
        const uint32_t x = compact3(ind), y = compact3(ind >> 1), z = compact3(ind >> 2);
        const float *g = tmp + (size_t)c * H3;
        float r = tmp[n];
        if (x + 1 < H) r = fmaxf(r, g[morton3(x + 1, y, z)]);
        if (x > 0) r = fmaxf(r, g[morton3(x - 1, y, z)]);
        if (y + 1 < H) r = fmaxf(r, g[morton3(x, y + 1, z)]);
        if (y > 0) r = fmaxf(r, g[morton3(x, y - 1, z)]);
        if (z + 1 < H) r = fmaxf(r, g[morton3(x, y, z + 1)]);
        if (z > 0) r = fmaxf(r, g[morton3(x, y, z - 1)]);
        float v = grid[n];
        if (v >= 0.f && r >= 0.f) {
            v = fmaxf(__fmul_rn(v, decay), r);
            grid[n] = v;
        }
        acc += (double)fmaxf(v, 0.f);
    }
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// radnerf_torso.py:235-241: tmp = max_pool2d(tmp, 5, stride 1, padding 2) (out-of-range cells are -inf: skipped);
// grid = max(grid * decay, tmp) everywhere (no untrained cells in the torso grid); then this block's share of sum(grid) in double
// (no clamp: the torso mean is a plain mean).  tmp and grid are [H, H]; the 5x5 window is symmetric in x and y.
__global__ void __launch_bounds__(RED_NT) k_torso_dilate_ema(const float *__restrict__ tmp, uint32_t H, float decay,
                                                             float *__restrict__ grid, double *__restrict__ partial) {
    __shared__ double sh[RED_NT / 32];
    const uint32_t total = H * H;
    double acc = 0.0;
    const uint32_t base = blockIdx.x * RED_CELLS;
    for (int k = 0; k < RED_PER_THREAD; ++k) {
        const uint32_t n = base + k * RED_NT + threadIdx.x;
        if (n >= total) break;
        const int y = (int)(n / H), x = (int)(n - (uint32_t)y * H), h = (int)H;
        float r = tmp[n];
        for (int yy = max(y - 2, 0); yy <= min(y + 2, h - 1); ++yy)
            for (int xx = max(x - 2, 0); xx <= min(x + 2, h - 1); ++xx) r = fmaxf(r, tmp[yy * h + xx]);
        const float v = fmaxf(__fmul_rn(grid[n], decay), r);
        grid[n] = v;
        acc += (double)v;
    }
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// mean = sum(partials) / count (one block, fixed order); threshold = min(mean, density_thresh) (renderer.py:272-276)
__global__ void __launch_bounds__(RED_NT) k_mean_thresh(const double *__restrict__ partial, uint32_t n_partial, uint32_t count,
                                                        float density_thresh, float *__restrict__ mean_out, float *__restrict__ thresh_out) {
    __shared__ double sh[RED_NT / 32];
    double acc = 0.0;
    for (uint32_t i = threadIdx.x; i < n_partial; i += RED_NT) acc += partial[i];
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) {
        const float mean = (float)(s / (double)count);
        *mean_out = mean;
        *thresh_out = fminf(mean, density_thresh);
    }
}

// raymarching.cu packbits with the threshold read on the device (no host round trip for the mean)
__global__ void k_packbits_dev(const float *__restrict__ grid, uint32_t N, const float *__restrict__ thresh_p, uint8_t *__restrict__ bitfield) {
    const float thresh = *thresh_p;
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        const float4 a = *reinterpret_cast<const float4 *>(grid + (size_t)n * 8), b = *reinterpret_cast<const float4 *>(grid + (size_t)n * 8 + 4);
        uint32_t bits = 0;
        bits |= a.x > thresh ? 1u : 0u; bits |= a.y > thresh ? 2u : 0u; bits |= a.z > thresh ? 4u : 0u; bits |= a.w > thresh ? 8u : 0u;
        bits |= b.x > thresh ? 16u : 0u; bits |= b.y > thresh ? 32u : 0u; bits |= b.z > thresh ? 64u : 0u; bits |= b.w > thresh ? 128u : 0u;
        bitfield[n] = (uint8_t)bits;
    }
}

// renderer.py:159-196, one thread per (cascade, cell): the cell is marked -1 when no camera's frustum test passes.
// poses [B,16] row-major c2w.  Same operation order as the reference's fp32 CPU arithmetic:
//   cam = (xyz - t) @ R;  z > 0  &&  |cam.x| < (cx/fx)*z + 2*hgs  &&  |cam.y| < (cy/fy)*z + 2*hgs
struct UntrainedArgs {
    const float *poses;
    uint32_t B, C, H;
    float rx, ry;                 // float(cx / fx), float(cy / fy)
    float cell_scale[8], pad[8];  // per cascade: float(bound_c - hgs_c), float(2 * hgs_c)
    float *grid;
};

__global__ void k_mark_untrained(const __grid_constant__ UntrainedArgs a) {
    const uint32_t H3 = a.H * a.H * a.H, total = a.C * H3;
    for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < total; n += gridDim.x * blockDim.x) {
        const uint32_t cas = n / H3, m = n - cas * H3;
        const uint32_t c[3] = {compact3(m), compact3(m >> 1), compact3(m >> 2)};
        float w[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            w[k] = __fmul_rn(__fsub_rn(__fdiv_rn(__fmul_rn(2.0f, (float)c[k]), (float)(a.H - 1)), 1.0f), a.cell_scale[cas]);
        const float pad = a.pad[cas];
        bool seen = false;
        for (uint32_t b = 0; b < a.B && !seen; ++b) {
            const float *P = a.poses + (size_t)b * 16;
            const float d0 = __fsub_rn(w[0], P[3]), d1 = __fsub_rn(w[1], P[7]), d2 = __fsub_rn(w[2], P[11]);
            float q[3];
#pragma unroll
            for (int j = 0; j < 3; ++j)
                q[j] = __fadd_rn(__fadd_rn(__fmul_rn(d0, P[j]), __fmul_rn(d1, P[4 + j])), __fmul_rn(d2, P[8 + j]));
            seen = q[2] > 0.f && fabsf(q[0]) < __fadd_rn(__fmul_rn(a.rx, q[2]), pad) && fabsf(q[1]) < __fadd_rn(__fmul_rn(a.ry, q[2]), pad);
        }
        if (!seen) a.grid[n] = -1.0f;
    }
}

}  // namespace

uint32_t dilate_ema_blocks(uint32_t C, uint32_t H) { return (C * H * H * H + RED_CELLS - 1) / RED_CELLS; }

cudaError_t launch_grid_refresh_tail(const float *tmp, uint32_t C, uint32_t H, float decay, float density_thresh, float *grid,
                                     double *partial, float *mean_out, float *thresh_dev, uint8_t *bitfield, int *n_launches, cudaStream_t st) {
    *n_launches = 0;
    const uint32_t nb = dilate_ema_blocks(C, H);
    k_dilate_ema<<<nb, RED_NT, 0, st>>>(tmp, C, H, decay, grid, partial);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ++*n_launches;
    k_mean_thresh<<<1, RED_NT, 0, st>>>(partial, nb, C * H * H * H, density_thresh, mean_out, thresh_dev);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ++*n_launches;
    const uint32_t nbytes = C * H * H * H / 8;
    k_packbits_dev<<<grid_for(nbytes, 256), 256, 0, st>>>(grid, nbytes, thresh_dev, bitfield);
    e = cudaGetLastError();
    if (e == cudaSuccess) ++*n_launches;
    return e;
}

uint32_t torso_dilate_ema_blocks(uint32_t H) { return (H * H + RED_CELLS - 1) / RED_CELLS; }

cudaError_t launch_torso_grid_tail(const float *tmp, uint32_t H, float decay, float density_thresh, float *grid, double *partial,
                                   float *mean_out, float *thresh_dev, int *n_launches, cudaStream_t st) {
    *n_launches = 0;
    const uint32_t nb = torso_dilate_ema_blocks(H);
    k_torso_dilate_ema<<<nb, RED_NT, 0, st>>>(tmp, H, decay, grid, partial);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ++*n_launches;
    k_mean_thresh<<<1, RED_NT, 0, st>>>(partial, nb, H * H, density_thresh, mean_out, thresh_dev);
    e = cudaGetLastError();
    if (e == cudaSuccess) ++*n_launches;
    return e;
}

cudaError_t launch_mark_untrained(const float *poses, uint32_t B, float rx, float ry, const float *cell_scale, const float *pad, uint32_t C,
                                  uint32_t H, float *grid, cudaStream_t st) {
    UntrainedArgs a;
    a.poses = poses; a.B = B; a.C = C; a.H = H; a.rx = rx; a.ry = ry; a.grid = grid;
    for (uint32_t c = 0; c < 8; ++c) { a.cell_scale[c] = c < C ? cell_scale[c] : 0.f; a.pad[c] = c < C ? pad[c] : 0.f; }
    k_mark_untrained<<<grid_for((uint64_t)C * H * H * H, 256), 256, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gfpp
