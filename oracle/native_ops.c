/*
 * oracle/native_ops.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, CPU, fp32 restatement of the native ops that sit under modules/radnerfs in
 * yerfor/GeneFacePlusPlus: the six inference ops and (second half of the file) the training-side ones.  The reference ships these ops as
 * CUDA only (its Python wrappers force .cuda()); there is no CPU implementation and
 * the reference has no tests or golden vectors for them, so this file is the CPU
 * checker ("oracle") that the GPU kernels are compared against.  It is pinned by
 *   (i)  the reference's own PyTorch modules driven on CPU through these functions
 *        (oracle/validate_against_reference.py, run where /root/reference exists), and
 *   (ii) the reference's own CUDA kernels compiled unmodified into oracle/_ref and
 *        run on the GPU (tests/test_gpu_ref_pin.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library.  The product path never does.
 *
 * Build: see oracle/Makefile.  MUST be compiled with -ffp-contract=off so that every
 * float expression below has exactly the source-level (unfused) rounding; the CUDA
 * kernels mirror the discrete decisions (cell index, occupancy, termination) with
 * explicit __fmul_rn/__fadd_rn for the same reason (SURVEY.md section 7, H2).
 *
 * Each function cites the reference file:line whose behaviour it follows
 * (paths relative to /root/reference).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API __attribute__((visibility("default")))

/* ---- small helpers (modules/radnerfs/raymarching/src/raymarching.cu:19-81) ---- */

static inline float clampf(float v, float lo, float hi) { return fminf(hi, fmaxf(lo, v)); }

static inline float sign1f(float v) { return copysignf(1.0f, v); }

/* raymarching.cu:43-48: exponent of max|coord| picks the cascade */
static inline int cascade_from_pos(float x, float y, float z, float n_cascade) {
    float m = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
    int e;
    (void)frexpf(m, &e);
    return (int)fminf(n_cascade - 1.0f, fmaxf(0.0f, (float)e));
}

/* raymarching.cu:50-55: note the product is evaluated in DOUBLE because of the 0.5
 * literal, then rounded to float on assignment. */
static inline int cascade_from_dt(float dt, float H, float n_cascade) {
    float m = (float)((double)(dt * H) * 0.5);
    int e;
    (void)frexpf(m, &e);
    return (int)fminf(n_cascade - 1.0f, fmaxf(0.0f, (float)e));
}

/* raymarching.cu:57-72: 10-bit-per-axis Morton interleave */
static inline uint32_t spread3(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
static inline uint32_t morton3(uint32_t x, uint32_t y, uint32_t z) {
    return spread3(x) | (spread3(y) << 1) | (spread3(z) << 2);
}

ORC_API void orc_morton3D(const int32_t *coords, uint32_t N, int32_t *indices) {
    /* raymarching.cu:214-232 */
    for (uint32_t n = 0; n < N; ++n)
        indices[n] = (int32_t)morton3((uint32_t)coords[3 * n], (uint32_t)coords[3 * n + 1],
                                      (uint32_t)coords[3 * n + 2]);
}

ORC_API void orc_packbits(const float *grid, uint32_t N, float density_thresh, uint8_t *bitfield) {
    /* raymarching.cu:267-300: bit i of byte n <- grid[8n+i] > thresh */
    for (uint32_t n = 0; n < N; ++n) {
        uint8_t b = 0;
        for (int i = 0; i < 8; ++i)
            if (grid[(size_t)n * 8 + i] > density_thresh) b |= (uint8_t)(1u << i);
        bitfield[n] = b;
    }
}

/* ---- near_far_from_aabb (raymarching.cu:91-145) ---- */
ORC_API void orc_near_far_from_aabb(const float *rays_o, const float *rays_d, const float *aabb,
                                    uint32_t N, float min_near, float *nears, float *fars) {
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        const float *o = rays_o + 3 * n, *d = rays_d + 3 * n;
        const float rdx = 1.0f / d[0], rdy = 1.0f / d[1], rdz = 1.0f / d[2];
        float tn = (aabb[0] - o[0]) * rdx, tf = (aabb[3] - o[0]) * rdx;
        if (tn > tf) { float s = tn; tn = tf; tf = s; }
        float tny = (aabb[1] - o[1]) * rdy, tfy = (aabb[4] - o[1]) * rdy;
        if (tny > tfy) { float s = tny; tny = tfy; tfy = s; }
        if (tn > tfy || tny > tf) { nears[n] = fars[n] = FLT_MAX; continue; }
        if (tny > tn) tn = tny;
        if (tfy < tf) tf = tfy;
        float tnz = (aabb[2] - o[2]) * rdz, tfz = (aabb[5] - o[2]) * rdz;
        if (tnz > tfz) { float s = tnz; tnz = tfz; tfz = s; }
        if (tn > tfz || tnz > tf) { nears[n] = fars[n] = FLT_MAX; continue; }
        if (tnz > tn) tn = tnz;
        if (tfz < tf) tf = tfz;
        if (tn < min_near) tn = min_near;
        nears[n] = tn;
        fars[n] = tf;
    }
}

/* ---- march_rays (raymarching.cu:827-929) ----
 * One call = one "round" of the host loop: for each alive ray emit up to n_step
 * occupied samples starting from rays_t[ray].  Outputs must be zero-initialised by the
 * caller (the Python wrapper does torch.zeros: raymarching.py:383-385); unwritten rows
 * (deltas == 0) mean "ray ran out". */
ORC_API void orc_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t *rays_alive,
                            const float *rays_t, const float *rays_o, const float *rays_d,
                            float bound, float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H,
                            const uint8_t *grid, const float *nears, const float *fars,
                            float *xyzs, float *dirs, float *deltas, const float *noises) {
    const float rH = 1.0f / (float)H;
    const float H3 = (float)(H * H * H);
    const float sqrt3 = 1.7320508075688772f;
    const float dt_max = 2 * sqrt3 * (float)(1 << (C - 1)) / (float)H;
    const float dt_min = fminf(dt_max, 2 * sqrt3 / (float)max_steps);
    const float Hm1 = (float)(H - 1);
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t n = 0; n < (int64_t)n_alive; ++n) {
        const int32_t ray = rays_alive[n];
        const float *o = rays_o + 3 * (size_t)ray, *d = rays_d + 3 * (size_t)ray;
        float *px = xyzs + (size_t)n * n_step * 3;
        float *pd = dirs + (size_t)n * n_step * 3;
        float *pl = deltas + (size_t)n * n_step * 2;
        const float ox = o[0], oy = o[1], oz = o[2];
        const float dx = d[0], dy = d[1], dz = d[2];
        const float rdx = 1.0f / dx, rdy = 1.0f / dy, rdz = 1.0f / dz;
        float t = rays_t[ray];
        const float far = fars[ray];
        (void)nears;
        uint32_t step = 0;
        t += clampf(t * dt_gamma, dt_min, dt_max) * noises[n];
        while (t < far && step < n_step) {
            const float x = clampf(ox + t * dx, -bound, bound);
            const float y = clampf(oy + t * dy, -bound, bound);
            const float z = clampf(oz + t * dz, -bound, bound);
            const float dt = clampf(t * dt_gamma, dt_min, dt_max);
            const int ca = cascade_from_pos(x, y, z, (float)C);
            const int cb = cascade_from_dt(dt, (float)H, (float)C);
            const int level = ca > cb ? ca : cb;
            const float mip_bound = fminf(scalbnf(1.0f, level), bound);
            const float mip_rbound = 1.0f / mip_bound;
            /* 0.5 * (x*rb + 1) * H is a double expression in the reference (0.5 literal) */
            const int nx = (int)clampf((float)(0.5 * (double)(x * mip_rbound + 1.0f) * (double)H), 0.0f, Hm1);
            const int ny = (int)clampf((float)(0.5 * (double)(y * mip_rbound + 1.0f) * (double)H), 0.0f, Hm1);
            const int nz = (int)clampf((float)(0.5 * (double)(z * mip_rbound + 1.0f) * (double)H), 0.0f, Hm1);
            /* bit index formed in float: level * H3 + morton (exact below 2^24) */
            const uint32_t bit = (uint32_t)((float)level * H3 + (float)morton3((uint32_t)nx, (uint32_t)ny, (uint32_t)nz));
            const int occ = grid[bit / 8] & (1 << (bit % 8));
            if (occ) {
                px[0] = x; px[1] = y; px[2] = z;
                pd[0] = dx; pd[1] = dy; pd[2] = dz;
                t += dt;
                pl[0] = dt; pl[1] = t;
                px += 3; pd += 3; pl += 2;
                ++step;
            } else {
                const float tx = ((((float)nx + 0.5f + 0.5f * sign1f(dx)) * rH * 2 - 1) * mip_bound - x) * rdx;
                const float ty = ((((float)ny + 0.5f + 0.5f * sign1f(dy)) * rH * 2 - 1) * mip_bound - y) * rdy;
                const float tz = ((((float)nz + 0.5f + 0.5f * sign1f(dz)) * rH * 2 - 1) * mip_bound - z) * rdz;
                const float tt = t + fmaxf(0.0f, fminf(tx, fminf(ty, tz)));
                do {
                    t += clampf(t * dt_gamma, dt_min, dt_max);
                } while (t < tt);
            }
        }
    }
}

/* ---- composite_rays (raymarching.cu:942-1029) ----
 * In place on weights_sum/depth/image/rays_t; kills rays by writing -1 into rays_alive.
 * The reference uses the approximate __expf; the oracle uses exact expf (SURVEY H6). */
ORC_API void orc_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t *rays_alive,
                                float *rays_t, const float *sigmas, const float *rgbs,
                                const float *deltas, float *weights_sum, float *depth, float *image) {
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)n_alive; ++n) {
        const int32_t ray = rays_alive[n];
        const float *sg = sigmas + (size_t)n * n_step;
        const float *cl = rgbs + (size_t)n * n_step * 3;
        const float *dl = deltas + (size_t)n * n_step * 2;
        float t = rays_t[ray];
        float ws = weights_sum[ray], dp = depth[ray];
        float r = image[3 * (size_t)ray], g = image[3 * (size_t)ray + 1], b = image[3 * (size_t)ray + 2];
        uint32_t step = 0;
        while (step < n_step) {
            if (dl[0] == 0) break;
            const float alpha = 1.0f - expf(-sg[0] * dl[0]);
            const float T = 1 - ws;
            const float w = alpha * T;
            ws += w;
            t = dl[1];
            dp += w * t;
            r += w * cl[0];
            g += w * cl[1];
            b += w * cl[2];
            if (T < T_thresh) break;
            ++sg; cl += 3; dl += 2; ++step;
        }
        if (step < n_step) rays_alive[n] = -1;
        else rays_t[ray] = t;
        weights_sum[ray] = ws;
        depth[ray] = dp;
        image[3 * (size_t)ray] = r;
        image[3 * (size_t)ray + 1] = g;
        image[3 * (size_t)ray + 2] = b;
    }
}

/* ---- grid_encode_forward (gridencoder.cu:50-84, 87-196; forward only, no dy_dx) ----
 * inputs [B,D] in [0,1]; embeddings [sum,Cc]; offsets [L+1]; outputs [L,B,Cc] (L-major). */
static inline uint32_t grid_index(uint32_t D, uint32_t Cc, uint32_t gridtype, int align_corners,
                                  uint32_t hashmap_size, uint32_t resolution, const uint32_t *pg) {
    static const uint32_t primes[7] = {1u, 2654435761u, 805459861u, 3674653429u,
                                       2097192037u, 1434869437u, 2165219737u};
    uint32_t stride = 1, index = 0;
    /* dimensions stop contributing once stride exceeds the level's table size (H5) */
    for (uint32_t d = 0; d < D && stride <= hashmap_size; ++d) {
        index += pg[d] * stride;
        stride *= align_corners ? resolution : (resolution + 1);
    }
    if (gridtype == 0 && stride > hashmap_size) {
        uint32_t h = 0;
        for (uint32_t d = 0; d < D; ++d) h ^= pg[d] * primes[d];
        index = h;
    }
    return (index % hashmap_size) * Cc;
}

ORC_API int orc_grid_encode_forward(const float *inputs, const float *embeddings, const int32_t *offsets,
                                    float *outputs, uint32_t B, uint32_t D, uint32_t Cc, uint32_t L,
                                    float S, uint32_t H, uint32_t gridtype, int align_corners,
                                    uint32_t interp) {
    if (D < 2 || D > 5) return -1;
    if (!(Cc == 1 || Cc == 2 || Cc == 4 || Cc == 8)) return -2;
    for (uint32_t level = 0; level < L; ++level) {
        const float *tab = embeddings + (size_t)(uint32_t)offsets[level] * Cc;
        const uint32_t hashmap_size = (uint32_t)(offsets[level + 1] - offsets[level]);
        const float scale = exp2f((float)level * S) * (float)H - 1.0f;
        const uint32_t resolution = (uint32_t)ceil((double)scale) + 1;
#pragma omp parallel for schedule(static)
        for (int64_t b = 0; b < (int64_t)B; ++b) {
            const float *in = inputs + (size_t)b * D;
            float *out = outputs + ((size_t)level * B + (size_t)b) * Cc;
            int oob = 0;
            for (uint32_t d = 0; d < D; ++d)
                if (in[d] < 0 || in[d] > 1) oob = 1;
            if (oob) {
                for (uint32_t c = 0; c < Cc; ++c) out[c] = 0;
                continue;
            }
            float pos[5];
            uint32_t pg[5];
            for (uint32_t d = 0; d < D; ++d) {
                pos[d] = in[d] * scale + (align_corners ? 0.0f : 0.5f);
                pg[d] = (uint32_t)floorf(pos[d]);
                pos[d] -= (float)pg[d];
                if (interp == 1) pos[d] = pos[d] * pos[d] * (3.0f - 2.0f * pos[d]);
            }
            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t corner = 0; corner < (1u << D); ++corner) {
                float w = 1;
                uint32_t pl[5];
                for (uint32_t d = 0; d < D; ++d) {
                    if ((corner & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                const uint32_t idx = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pl);
                for (uint32_t c = 0; c < Cc; ++c) acc[c] += w * tab[idx + c];
            }
            for (uint32_t c = 0; c < Cc; ++c) out[c] = acc[c];
        }
    }
    return 0;
}

/* ---- sh_encode_forward (shencoder.cu:27-68; degree <= 4 is all the path uses) ---- */
ORC_API int orc_sh_encode_forward(const float *inputs, float *outputs, uint32_t B, uint32_t degree) {
    if (degree < 1 || degree > 4) return -1;
    const uint32_t C2 = degree * degree;
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < (int64_t)B; ++b) {
        const float x = inputs[3 * b], y = inputs[3 * b + 1], z = inputs[3 * b + 2];
        float *o = outputs + (size_t)b * C2;
        const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
        o[0] = 0.28209479177387814f;
        if (degree <= 1) continue;
        o[1] = -0.48860251190291987f * y;
        o[2] = 0.48860251190291987f * z;
        o[3] = -0.48860251190291987f * x;
        if (degree <= 2) continue;
        o[4] = 1.0925484305920792f * xy;
        o[5] = -1.0925484305920792f * yz;
        o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
        o[7] = -1.0925484305920792f * xz;
        o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
        if (degree <= 3) continue;
        o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
        o[10] = 2.8906114426405538f * xy * z;
        o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
        o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
        o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
        o[14] = 1.4453057213202769f * z * (x2 - y2);
        o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
    }
    return 0;
}

/* ---- freq_encode_forward (freqencoder.cu:30-58) ----
 * out[b] = [x_0..x_{D-1}, then for f<deg: sin(2^f x_d), sin(2^f x_d + pi/2)].
 * Reference uses __sinf; the oracle uses exact sinf (SURVEY H6). */
ORC_API void orc_freq_encode_forward(const float *inputs, uint32_t B, uint32_t D, uint32_t deg,
                                     uint32_t C, float *outputs) {
    const float half_pi = 3.141592653589793f / 2;
    (void)deg;
#pragma omp parallel for schedule(static)
    for (int64_t b = 0; b < (int64_t)B; ++b) {
        const float *in = inputs + (size_t)b * D;
        float *o = outputs + (size_t)b * C;
        for (uint32_t c = 0; c < C; ++c) {
            if (c < D) { o[c] = in[c]; continue; }
            const uint32_t col = c / D - 1, d = c % D, f = col / 2;
            const float phase = (float)(col % 2) * half_pi;
            o[c] = sinf(scalbnf(in[d], (int)f) + phase);
        }
    }
}

/* ---- bias-free Linear (+ optional ReLU) used by the three tiny MLPs ----
 * modules/radnerfs/cond_encoder.py:183-202 (nn.Linear(bias=False), ReLU between layers).
 * y[M,N] = x[M,K] @ W[N,K]^T, fp32 with a fixed k-ascending summation per output.
 * Used by the self-contained CPU baseline (oracle/render.py can also use torch's
 * F.linear; the two differ only by fp32 summation order). */
ORC_API void orc_linear(const float *x, const float *W, float *y, uint32_t M, uint32_t K, uint32_t N,
                        int relu) {
#pragma omp parallel for schedule(static)
    for (int64_t m = 0; m < (int64_t)M; ++m) {
        const float *xr = x + (size_t)m * K;
        float *yr = y + (size_t)m * N;
        for (uint32_t n = 0; n < N; ++n) {
            const float *wr = W + (size_t)n * K;
            float acc = 0;
            for (uint32_t k = 0; k < K; ++k) acc += xr[k] * wr[k];
            yr[n] = (relu && acc < 0) ? 0.0f : acc;
        }
    }
}

/* ==================================================================================================
 * Training-side ops (SURVEY.md 8(f) rank 4): CPU restatement of the reference's training kernels.
 * Parity of these is pinned on the GPU against the reference's own kernels (tests/test_gpu_ref_pin.py).
 * ================================================================================================== */

/* one marching pass of kernel_march_rays_train (raymarching.cu:397-443 count, :464-517 write): walks ray n from t0 and
 * returns the number of occupied samples (<= limit); when px != NULL it also writes them. */
static uint32_t march_train_pass(const float *o, const float *d, const uint8_t *grid, float bound, float dt_gamma,
                                 float dt_min, float dt_max, uint32_t C, uint32_t H, float t0, float far, uint32_t limit,
                                 float *px, float *pd, float *pl) {
    const float rH = 1.0f / (float)H, H3 = (float)(H * H * H), Hm1 = (float)(H - 1);
    const float ox = o[0], oy = o[1], oz = o[2], dx = d[0], dy = d[1], dz = d[2];
    const float rdx = 1.0f / dx, rdy = 1.0f / dy, rdz = 1.0f / dz;
    float t = t0;
    uint32_t step = 0;
    while (t < far && step < limit) {
        const float x = clampf(ox + t * dx, -bound, bound);
        const float y = clampf(oy + t * dy, -bound, bound);
        const float z = clampf(oz + t * dz, -bound, bound);
        const float dt = clampf(t * dt_gamma, dt_min, dt_max);
        const int ca = cascade_from_pos(x, y, z, (float)C);
        const int cb = cascade_from_dt(dt, (float)H, (float)C);
        const int level = ca > cb ? ca : cb;
        const float mip_bound = fminf(scalbnf(1.0f, level), bound);
        const float mip_rbound = 1.0f / mip_bound;
        const int nx = (int)clampf((float)(0.5 * (double)(x * mip_rbound + 1.0f) * (double)H), 0.0f, Hm1);
        const int ny = (int)clampf((float)(0.5 * (double)(y * mip_rbound + 1.0f) * (double)H), 0.0f, Hm1);
        const int nz = (int)clampf((float)(0.5 * (double)(z * mip_rbound + 1.0f) * (double)H), 0.0f, Hm1);
        const uint32_t bit = (uint32_t)((float)level * H3 + (float)morton3((uint32_t)nx, (uint32_t)ny, (uint32_t)nz));
        const int occ = grid[bit / 8] & (1 << (bit % 8));
        if (occ) {
            if (px) {
                px[0] = x; px[1] = y; px[2] = z;
                pd[0] = dx; pd[1] = dy; pd[2] = dz;
                pl[0] = dt; pl[1] = t + dt;
                px += 3; pd += 3; pl += 2;
            }
            t += dt;
            ++step;
        } else {
            const float tx = ((((float)nx + 0.5f + 0.5f * sign1f(dx)) * rH * 2 - 1) * mip_bound - x) * rdx;
            const float ty = ((((float)ny + 0.5f + 0.5f * sign1f(dy)) * rH * 2 - 1) * mip_bound - y) * rdy;
            const float tz = ((((float)nz + 0.5f + 0.5f * sign1f(dz)) * rH * 2 - 1) * mip_bound - z) * rdz;
            const float tt = t + fmaxf(0.0f, fminf(tx, fminf(ty, tz)));
            do {
                t += clampf(t * dt_gamma, dt_min, dt_max);
            } while (t < tt);
        }
    }
    return step;
}

/* ---- march_rays_train (raymarching.cu:352-533) ----
 * The reference hands out point offsets with atomicAdd in whatever order the threads arrive (:445-446), so its layout is
 * non-deterministic; the per-ray CONTENT (rays[i] = (ray, offset, num_steps) and the samples at that offset) is what is
 * defined.  The oracle assigns offsets in ray order (exclusive prefix sum of the counts) and rays[n] = (n, offset, steps):
 * one of the layouts the reference can produce.  counter[0] += total points, counter[1] += N.  Rays whose samples would
 * overflow M keep their `rays` row but write nothing (:455-456). */
ORC_API void orc_march_rays_train(const float *rays_o, const float *rays_d, const uint8_t *grid, float bound, float dt_gamma,
                                  uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float *nears,
                                  const float *fars, float *xyzs, float *dirs, float *deltas, int32_t *rays, int32_t *counter,
                                  const float *noises) {
    const float sqrt3 = 1.7320508075688772f;
    const float dt_max = 2 * sqrt3 * (float)(1 << (C - 1)) / (float)H;
    const float dt_min = fminf(dt_max, 2 * sqrt3 / (float)max_steps);
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        float t0 = nears[n];
        t0 += clampf(t0 * dt_gamma, dt_min, dt_max) * noises[n];
        rays[3 * n] = (int32_t)n;
        rays[3 * n + 2] = (int32_t)march_train_pass(rays_o + 3 * n, rays_d + 3 * n, grid, bound, dt_gamma, dt_min, dt_max, C, H, t0,
                                                    fars[n], max_steps, 0, 0, 0);
    }
    uint32_t off = (uint32_t)counter[0];
    for (uint32_t n = 0; n < N; ++n) { rays[3 * n + 1] = (int32_t)off; off += (uint32_t)rays[3 * n + 2]; }
    counter[0] = (int32_t)off;
    counter[1] += (int32_t)N;
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        const uint32_t ns = (uint32_t)rays[3 * n + 2], po = (uint32_t)rays[3 * n + 1];
        if (ns == 0 || po + ns > M) continue;
        float t0 = nears[n];
        t0 += clampf(t0 * dt_gamma, dt_min, dt_max) * noises[n];
        march_train_pass(rays_o + 3 * n, rays_d + 3 * n, grid, bound, dt_gamma, dt_min, dt_max, C, H, t0, fars[n], ns,
                         xyzs + 3 * (size_t)po, dirs + 3 * (size_t)po, deltas + 2 * (size_t)po);
    }
}

/* ---- march_rays_train_backward (raymarching.cu:535-598): xyz = o + t d with t = deltas[.,1] ---- */
ORC_API void orc_march_rays_train_backward(const float *grad_xyzs, const float *grad_dirs, const int32_t *rays, const float *deltas,
                                           uint32_t N, uint32_t M, float *grad_rays_o, float *grad_rays_d) {
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        /* NOTE the reference indexes grad_rays_* by the thread id n, not by rays[n].index (:548-549) */
        const uint32_t off = (uint32_t)rays[3 * n + 1], ns = (uint32_t)rays[3 * n + 2];
        if (ns == 0 || off + ns > M) continue;
        float *go = grad_rays_o + 3 * n, *gd = grad_rays_d + 3 * n;
        for (uint32_t s = 0; s < ns; ++s) {
            const float *gx = grad_xyzs + 3 * (size_t)(off + s), *gdd = grad_dirs + 3 * (size_t)(off + s);
            const float t = deltas[2 * (size_t)(off + s) + 1];
            for (int c = 0; c < 3; ++c) {
                go[c] += gx[c];
                gd[c] += gx[c] * t + gdd[c];
            }
        }
    }
}

/* ---- composite_rays_train_forward (raymarching.cu:603-700); exact expf instead of __expf (SURVEY H6) ---- */
ORC_API void orc_composite_rays_train_forward(const float *sigmas, const float *rgbs, const float *ambient, const float *deltas,
                                              const int32_t *rays, uint32_t M, uint32_t N, float T_thresh, float *weights_sum,
                                              float *ambient_sum, float *depth, float *image) {
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        const uint32_t index = (uint32_t)rays[3 * n], off = (uint32_t)rays[3 * n + 1], ns = (uint32_t)rays[3 * n + 2];
        float T = 1.0f, r = 0, g = 0, b = 0, ws = 0, dp = 0, amb = 0;
        if (!(ns == 0 || off + ns > M)) {
            for (uint32_t s = 0; s < ns; ++s) {
                const size_t i = (size_t)off + s;
                const float alpha = 1.0f - expf(-sigmas[i] * deltas[2 * i]);
                const float w = alpha * T;
                r += w * rgbs[3 * i]; g += w * rgbs[3 * i + 1]; b += w * rgbs[3 * i + 2];
                dp += w * deltas[2 * i + 1];
                ws += w;
                amb += ambient[i];
                T *= 1.0f - alpha;
                if (T < T_thresh) break;
            }
        }
        weights_sum[index] = ws; ambient_sum[index] = amb; depth[index] = dp;
        image[3 * (size_t)index] = r; image[3 * (size_t)index + 1] = g; image[3 * (size_t)index + 2] = b;
    }
}

/* ---- composite_rays_train_backward (raymarching.cu:711-822) ----
 * grad_* outputs must be zero-initialised by the caller (the wrapper does torch.zeros_like, raymarching.py:316-318):
 * samples after the T_thresh cut keep 0. */
ORC_API void orc_composite_rays_train_backward(const float *grad_weights_sum, const float *grad_ambient_sum, const float *grad_image,
                                               const float *sigmas, const float *rgbs, const float *ambient, const float *deltas,
                                               const int32_t *rays, const float *weights_sum, const float *ambient_sum,
                                               const float *image, uint32_t M, uint32_t N, float T_thresh, float *grad_sigmas,
                                               float *grad_rgbs, float *grad_ambient) {
    (void)ambient; (void)ambient_sum;
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        const uint32_t index = (uint32_t)rays[3 * n], off = (uint32_t)rays[3 * n + 1], ns = (uint32_t)rays[3 * n + 2];
        if (ns == 0 || off + ns > M) continue;
        const float *gi = grad_image + 3 * (size_t)index;
        const float gws = grad_weights_sum[index], gamb = grad_ambient_sum[index];
        const float rf = image[3 * (size_t)index], gf = image[3 * (size_t)index + 1], bf = image[3 * (size_t)index + 2];
        const float wsf = weights_sum[index];
        float T = 1.0f, r = 0, g = 0, b = 0, ws = 0;
        for (uint32_t s = 0; s < ns; ++s) {
            const size_t i = (size_t)off + s;
            const float alpha = 1.0f - expf(-sigmas[i] * deltas[2 * i]);
            const float w = alpha * T;
            r += w * rgbs[3 * i]; g += w * rgbs[3 * i + 1]; b += w * rgbs[3 * i + 2];
            ws += w;
            T *= 1.0f - alpha;
            grad_rgbs[3 * i] = gi[0] * w; grad_rgbs[3 * i + 1] = gi[1] * w; grad_rgbs[3 * i + 2] = gi[2] * w;
            grad_ambient[i] = gamb;
            grad_sigmas[i] = deltas[2 * i] * (gi[0] * (T * rgbs[3 * i] - (rf - r)) + gi[1] * (T * rgbs[3 * i + 1] - (gf - g)) +
                                              gi[2] * (T * rgbs[3 * i + 2] - (bf - b)) + gws * (1 - wsf));
            if (T < T_thresh) break;
        }
        (void)ws;
    }
}

/* ---- grid encoder: dy_dx of the forward (gridencoder.cu:198-243), [B, L, D, Cc] ---- */
ORC_API int orc_grid_encode_dydx(const float *inputs, const float *embeddings, const int32_t *offsets, float *dy_dx, uint32_t B,
                                 uint32_t D, uint32_t Cc, uint32_t L, float S, uint32_t H, uint32_t gridtype, int align_corners,
                                 uint32_t interp) {
    if (D < 2 || D > 5 || Cc > 8) return -1;
    for (uint32_t level = 0; level < L; ++level) {
        const float *tab = embeddings + (size_t)(uint32_t)offsets[level] * Cc;
        const uint32_t hashmap_size = (uint32_t)(offsets[level + 1] - offsets[level]);
        const float scale = exp2f((float)level * S) * (float)H - 1.0f;
        const uint32_t resolution = (uint32_t)ceil((double)scale) + 1;
#pragma omp parallel for schedule(static)
        for (int64_t b = 0; b < (int64_t)B; ++b) {
            const float *in = inputs + (size_t)b * D;
            float *out = dy_dx + ((size_t)b * L + level) * D * Cc;
            int oob = 0;
            for (uint32_t d = 0; d < D; ++d)
                if (in[d] < 0 || in[d] > 1) oob = 1;
            if (oob) {   /* :126-134 zeroes dy_dx for out-of-range inputs */
                for (uint32_t i = 0; i < D * Cc; ++i) out[i] = 0;
                continue;
            }
            float pos[5], deriv[5];
            uint32_t pg[5];
            for (uint32_t d = 0; d < D; ++d) {
                pos[d] = in[d] * scale + (align_corners ? 0.0f : 0.5f);
                pg[d] = (uint32_t)floorf(pos[d]);
                pos[d] -= (float)pg[d];
                if (interp == 1) { deriv[d] = 6 * pos[d] * (1 - pos[d]); pos[d] = pos[d] * pos[d] * (3.0f - 2.0f * pos[d]); }
                else deriv[d] = 1.0f;
            }
            for (uint32_t gd = 0; gd < D; ++gd) {
                float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
                    float w = scale;
                    uint32_t pl[5];
                    for (uint32_t nd = 0; nd < D - 1; ++nd) {
                        const uint32_t d = nd >= gd ? nd + 1 : nd;
                        if ((idx & (1u << nd)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                        else { w *= pos[d]; pl[d] = pg[d] + 1; }
                    }
                    pl[gd] = pg[gd];
                    const uint32_t il = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pl);
                    pl[gd] = pg[gd] + 1;
                    const uint32_t ir = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pl);
                    for (uint32_t c = 0; c < Cc; ++c) acc[c] += w * (tab[ir + c] - tab[il + c]) * deriv[gd];
                }
                for (uint32_t c = 0; c < Cc; ++c) out[gd * Cc + c] = acc[c];
            }
        }
    }
    return 0;
}

/* ---- grid_encode_backward (gridencoder.cu:246-340 scatter into the table, :343-368 input gradient) ----
 * grad [L,B,Cc]; grad_embeddings accumulates (caller zero-initialises, grid.py:76); grad_inputs [B,D] is written when dy_dx
 * is given.  Sequential accumulation in b order (the reference's atomicAdd order is arbitrary). */
ORC_API int orc_grid_encode_backward(const float *grad, const float *inputs, const int32_t *offsets, float *grad_embeddings,
                                     uint32_t B, uint32_t D, uint32_t Cc, uint32_t L, float S, uint32_t H, const float *dy_dx,
                                     float *grad_inputs, uint32_t gridtype, int align_corners, uint32_t interp) {
    if (D < 2 || D > 5 || Cc > 8) return -1;
#pragma omp parallel for schedule(static)
    for (int64_t level = 0; level < (int64_t)L; ++level) {
        float *gt = grad_embeddings + (size_t)(uint32_t)offsets[level] * Cc;
        const uint32_t hashmap_size = (uint32_t)(offsets[level + 1] - offsets[level]);
        const float scale = exp2f((float)level * S) * (float)H - 1.0f;
        const uint32_t resolution = (uint32_t)ceil((double)scale) + 1;
        for (uint32_t b = 0; b < B; ++b) {
            const float *in = inputs + (size_t)b * D;
            const float *g = grad + ((size_t)level * B + b) * Cc;
            int oob = 0;
            for (uint32_t d = 0; d < D; ++d)
                if (in[d] < 0 || in[d] > 1) oob = 1;
            if (oob) continue;
            float pos[5];
            uint32_t pg[5];
            for (uint32_t d = 0; d < D; ++d) {
                pos[d] = in[d] * scale + (align_corners ? 0.0f : 0.5f);
                pg[d] = (uint32_t)floorf(pos[d]);
                pos[d] -= (float)pg[d];
                if (interp == 1) pos[d] = pos[d] * pos[d] * (3.0f - 2.0f * pos[d]);
            }
            for (uint32_t corner = 0; corner < (1u << D); ++corner) {
                float w = 1;
                uint32_t pl[5];
                for (uint32_t d = 0; d < D; ++d) {
                    if ((corner & (1u << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                const uint32_t idx = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pl);
                for (uint32_t c = 0; c < Cc; ++c) gt[idx + c] += w * g[c];
            }
        }
    }
    if (dy_dx && grad_inputs) {
#pragma omp parallel for schedule(static)
        for (int64_t t = 0; t < (int64_t)B * D; ++t) {
            const uint32_t b = (uint32_t)(t / D), d = (uint32_t)(t % D);
            const float *dd = dy_dx + (size_t)b * L * D * Cc;
            float r = 0;
            for (uint32_t l = 0; l < L; ++l)
                for (uint32_t c = 0; c < Cc; ++c) r += grad[((size_t)l * B + b) * Cc + c] * dd[(size_t)l * D * Cc + d * Cc + c];
            grad_inputs[t] = r;
        }
    }
    return 0;
}

/* ---- grad_total_variation (gridencoder.cu:505-592): adds the TV gradient of the cells the inputs fall in ---- */
ORC_API int orc_grad_total_variation(const float *inputs, const float *embeddings, float *grad, const int32_t *offsets, float weight,
                                     uint32_t B, uint32_t D, uint32_t Cc, uint32_t L, float S, uint32_t H, uint32_t gridtype,
                                     int align_corners) {
    if (D < 2 || D > 5 || Cc > 8) return -1;
#pragma omp parallel for schedule(static)
    for (int64_t level = 0; level < (int64_t)L; ++level) {
        const float *tab = embeddings + (size_t)(uint32_t)offsets[level] * Cc;
        float *gt = grad + (size_t)(uint32_t)offsets[level] * Cc;
        const uint32_t hashmap_size = (uint32_t)(offsets[level + 1] - offsets[level]);
        const float scale = exp2f((float)level * S) * (float)H - 1.0f;
        const uint32_t resolution = (uint32_t)ceil((double)scale) + 1;
        const float w = weight / (float)(2 * D);
        for (uint32_t b = 0; b < B; ++b) {
            const float *in = inputs + (size_t)b * D;
            int oob = 0;
            for (uint32_t d = 0; d < D; ++d)
                if (in[d] < 0 || in[d] > 1) oob = 1;
            if (oob) continue;
            uint32_t pg[5];
            for (uint32_t d = 0; d < D; ++d) pg[d] = (uint32_t)floorf(in[d] * scale + (align_corners ? 0.0f : 0.5f));
            float res[8] = {0, 0, 0, 0, 0, 0, 0, 0}, idelta[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const uint32_t index = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pg);
            for (uint32_t d = 0; d < D; ++d) {
                const uint32_t cur = pg[d];
                if (cur < resolution) {
                    pg[d] = cur + 1;
                    const uint32_t ir = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pg);
                    for (uint32_t c = 0; c < Cc; ++c) { const float gv = tab[index + c] - tab[ir + c]; res[c] += gv; idelta[c] += gv * gv; }
                }
                if (cur > 0) {
                    pg[d] = cur - 1;
                    const uint32_t il = grid_index(D, Cc, gridtype, align_corners, hashmap_size, resolution, pg);
                    for (uint32_t c = 0; c < Cc; ++c) { const float gv = tab[index + c] - tab[il + c]; res[c] += gv; idelta[c] += gv * gv; }
                }
                pg[d] = cur;
            }
            for (uint32_t c = 0; c < Cc; ++c) gt[index + c] += w * res[c] * (1.0f / sqrtf(idelta[c] + 1e-9f));
        }
    }
    return 0;
}

/* ---- update_extra_state helpers (raymarching.cu:237-262 invert, :303-342 dilation, :162-208 sph_from_ray) ---- */
static inline uint32_t compact3(uint32_t x) {
    x &= 0x49249249u;
    x = (x | (x >> 2)) & 0xC30C30C3u;
    x = (x | (x >> 4)) & 0x0F00F00Fu;
    x = (x | (x >> 8)) & 0xFF0000FFu;
    x = (x | (x >> 16)) & 0x0000FFFFu;
    return x;
}

ORC_API void orc_morton3D_invert(const int32_t *indices, uint32_t N, int32_t *coords) {
    for (uint32_t n = 0; n < N; ++n) {
        const uint32_t ind = (uint32_t)indices[n];
        coords[3 * n] = (int32_t)compact3(ind);
        coords[3 * n + 1] = (int32_t)compact3(ind >> 1);
        coords[3 * n + 2] = (int32_t)compact3(ind >> 2);
    }
}

ORC_API void orc_morton3D_dilation(const float *grid, uint32_t C, uint32_t H, float *out) {
    const uint32_t H3 = H * H * H;
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)C * H3; ++n) {
        const uint32_t c = (uint32_t)(n / H3), ind = (uint32_t)(n - (int64_t)c * H3);
        const uint32_t x = compact3(ind), y = compact3(ind >> 1), z = compact3(ind >> 2);
        const float *g = grid + (size_t)c * H3;
        float r = grid[n];
        if (x + 1 < H) r = fmaxf(r, g[morton3(x + 1, y, z)]);
        if (x > 0) r = fmaxf(r, g[morton3(x - 1, y, z)]);
        if (y + 1 < H) r = fmaxf(r, g[morton3(x, y + 1, z)]);
        if (y > 0) r = fmaxf(r, g[morton3(x, y - 1, z)]);
        if (z + 1 < H) r = fmaxf(r, g[morton3(x, y, z + 1)]);
        if (z > 0) r = fmaxf(r, g[morton3(x, y, z - 1)]);
        out[n] = r;
    }
}

ORC_API void orc_sph_from_ray(const float *rays_o, const float *rays_d, float radius, uint32_t N, float *coords) {
    const float rpi = 0.3183098861837907f;
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < (int64_t)N; ++n) {
        const float ox = rays_o[3 * n], oy = rays_o[3 * n + 1], oz = rays_o[3 * n + 2];
        const float dx = rays_d[3 * n], dy = rays_d[3 * n + 1], dz = rays_d[3 * n + 2];
        const float A = dx * dx + dy * dy + dz * dz;
        const float Bq = ox * dx + oy * dy + oz * dz;
        const float Cq = ox * ox + oy * oy + oz * oz - radius * radius;
        const float t = (-Bq + sqrtf(Bq * Bq - A * Cq)) / A;
        const float x = ox + t * dx, y = oy + t * dy, z = oz + t * dz;
        const float theta = atan2f(sqrtf(x * x + z * z), y);
        const float phi = atan2f(z, x);
        coords[2 * n] = 2 * theta * rpi - 1;
        coords[2 * n + 1] = phi * rpi;
    }
}

ORC_API void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

ORC_API int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
