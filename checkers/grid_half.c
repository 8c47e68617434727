/* checkers/grid_half.c -- TEST INFRASTRUCTURE: plain-C restatement of the grid encoder on half tables, the reference's
 * scalar_t = at::Half instantiations of kernel_grid, kernel_grid_backward and kernel_input_backward (gridencoder.cu:87-368),
 * for C = 2, D in {2,3}.  Built with -ffp-contract=off: every fp32 operation rounds where the source says, except the two
 * contractions the reference's SASS forms (scale = exp2f(l * S) * H - 1 and pos = x * scale + off), written here with fmaf.
 *
 * `rnd` selects the arithmetic: 1 = IEEE binary16 round-to-nearest-even at every site where at::Half rounds (the half kernels'
 * contract), 0 = the same expressions in fp32 with no 16-bit rounding (the reference's float instantiation), so that the two can
 * be compared site by site.  Tables and upstream gradients come in as fp32 arrays holding binary16 values.
 *
 * Level scales: scales[L] if given (the device exp2f values, for bit-exact comparisons with GPU kernels), else the host exp2f.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* ---- binary16 <-> fp32, round to nearest even ---- */
static float h2f(uint16_t h) {
    const uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
    uint32_t bits;
    if (e == 0) {
        const float v = (float)m * 5.9604644775390625e-8f;   /* m * 2^-24, exact */
        return s ? -v : v;
    }
    bits = e == 31 ? (s | 0x7f800000u | (m << 13)) : (s | ((e + 112u) << 23) | (m << 13));
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

static uint16_t f2h(float f) {
    uint32_t x;
    memcpy(&x, &f, 4);
    const uint32_t s = (x >> 16) & 0x8000u, a = x & 0x7fffffffu;
    if (a > 0x7f800000u) return (uint16_t)(s | 0x7e00u);             /* NaN */
    if (a >= 0x47800000u) return (uint16_t)(s | 0x7c00u);            /* >= 2^16: inf */
    if (a < 0x38800000u) {                                            /* below 2^-14: subnormal or zero, in units of 2^-24 */
        float v;
        memcpy(&v, &a, 4);
        return (uint16_t)(s | (uint32_t)rintf(v * 16777216.0f));     /* exact scaling, rintf rounds half to even */
    }
    /* normal: rebias the exponent and round the 13 dropped bits to nearest even (a carry may reach inf, as it should) */
    return (uint16_t)(s | ((a - 0x38000000u + 0xfffu + ((a >> 13) & 1u)) >> 13));
}

/* the value a rounding site leaves: binary16 in half mode, unchanged in fp32 mode */
static float R(float v, int rnd) { return rnd ? h2f(f2h(v)) : v; }

float ghc_round_half(float v) { return h2f(f2h(v)); }

typedef struct {
    float scale;
    uint32_t res, hs, off;
} level_t;

static level_t level_of(const int32_t *offsets, uint32_t l, float S, uint32_t H, const float *scales) {
    level_t v;
    v.off = (uint32_t)offsets[l];
    v.hs = (uint32_t)(offsets[l + 1] - offsets[l]);
    v.scale = scales ? scales[l] : fmaf(exp2f((float)l * S), (float)H, -1.0f);
    v.res = (uint32_t)ceilf(v.scale) + 1;
    return v;
}

static uint32_t slot_of(uint32_t D, uint32_t gridtype, int align, const level_t *lv, const uint32_t *p) {
    static const uint32_t primes[3] = {1u, 2654435761u, 805459861u};
    uint32_t stride = 1, index = 0, d;
    for (d = 0; d < D && stride <= lv->hs; ++d) {
        index += p[d] * stride;
        stride *= align ? lv->res : lv->res + 1;
    }
    if (gridtype == 0 && stride > lv->hs) {
        index = 0;
        for (d = 0; d < D; ++d) index ^= p[d] * primes[d];
    }
    return index % lv->hs;
}

static int cell_of(uint32_t D, const float *in, const level_t *lv, int align, uint32_t interp, uint32_t *pg, float *pos, float *deriv) {
    uint32_t d;
    for (d = 0; d < D; ++d)
        if (in[d] < 0.f || in[d] > 1.f) return 0;
    for (d = 0; d < D; ++d) {
        float p = fmaf(in[d], lv->scale, align ? 0.0f : 0.5f);
        pg[d] = (uint32_t)floorf(p);
        p -= (float)pg[d];
        if (interp == 1) {
            deriv[d] = (6.0f * p) * (1.0f - p);
            p = (p * p) * (3.0f - 2.0f * p);
        } else {
            deriv[d] = 1.0f;
        }
        pos[d] = p;
    }
    return 1;
}

/* corner idx of the 2^D cell: weight and integer position */
static float corner(uint32_t D, uint32_t idx, const uint32_t *pg, const float *pos, uint32_t *pl) {
    float w = 1.0f;
    uint32_t d;
    for (d = 0; d < D; ++d) {
        if ((idx & (1u << d)) == 0) { w *= 1.0f - pos[d]; pl[d] = pg[d]; }
        else { w *= pos[d]; pl[d] = pg[d] + 1; }
    }
    return w;
}

/* forward: outputs [L,B,2], dy_dx [B,L,D,2] or NULL; emb [entries,2] */
int ghc_forward(const float *inputs, const float *emb, const int32_t *offsets, uint32_t B, uint32_t D, uint32_t L, float S, uint32_t H,
                uint32_t gridtype, int align, uint32_t interp, const float *scales, int rnd, float *outputs, float *dy_dx) {
    if ((D != 2 && D != 3) || L == 0 || L > 16) return -1;
    for (uint32_t l = 0; l < L; ++l) {
        const level_t lv = level_of(offsets, l, S, H, scales);
        const float *tb = emb + 2 * (size_t)lv.off;
        for (uint32_t b = 0; b < B; ++b) {
            const float *in = inputs + (size_t)b * D;
            float *out = outputs + ((size_t)l * B + b) * 2;
            float *dd = dy_dx ? dy_dx + ((size_t)b * L + l) * D * 2 : 0;
            uint32_t pg[3], pl[3];
            float pos[3], deriv[3];
            if (!cell_of(D, in, &lv, align, interp, pg, pos, deriv)) {
                out[0] = out[1] = 0.f;
                if (dd) for (uint32_t i = 0; i < 2 * D; ++i) dd[i] = 0.f;
                continue;
            }
            float r0 = 0.f, r1 = 0.f;
            for (uint32_t idx = 0; idx < (1u << D); ++idx) {
                const float w = corner(D, idx, pg, pos, pl);
                const float *v = tb + 2 * (size_t)slot_of(D, gridtype, align, &lv, pl);
                r0 = R(r0 + R(w * v[0], rnd), rnd);
                r1 = R(r1 + R(w * v[1], rnd), rnd);
            }
            out[0] = r0;
            out[1] = r1;
            if (!dd) continue;
            for (uint32_t gd = 0; gd < D; ++gd) {
                float a0 = 0.f, a1 = 0.f;
                for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
                    float w = lv.scale;
                    for (uint32_t nd = 0; nd < D - 1; ++nd) {
                        const uint32_t d = nd >= gd ? nd + 1 : nd;
                        if ((idx & (1u << nd)) == 0) { w *= 1.0f - pos[d]; pl[d] = pg[d]; }
                        else { w *= pos[d]; pl[d] = pg[d] + 1; }
                    }
                    pl[gd] = pg[gd];
                    const float *lf = tb + 2 * (size_t)slot_of(D, gridtype, align, &lv, pl);
                    pl[gd] = pg[gd] + 1;
                    const float *rg = tb + 2 * (size_t)slot_of(D, gridtype, align, &lv, pl);
                    a0 = R(a0 + R((w * R(rg[0] - lf[0], rnd)) * deriv[gd], rnd), rnd);
                    a1 = R(a1 + R((w * R(rg[1] - lf[1], rnd)) * deriv[gd], rnd), rnd);
                }
                dd[2 * gd] = a0;
                dd[2 * gd + 1] = a1;
            }
        }
    }
    return 0;
}

/* table gradient as the exact (float64) sum of the terms each add rounds: sum [entries,2], abs_sum [entries,2] = sum of |term|,
 * count [entries] = number of adds into each entry (both channels get the same) */
int ghc_table_grad(const float *grad, const float *inputs, const int32_t *offsets, uint32_t B, uint32_t D, uint32_t L, float S, uint32_t H,
                   uint32_t gridtype, int align, uint32_t interp, const float *scales, int rnd, double *sum, double *abs_sum, int32_t *count) {
    if ((D != 2 && D != 3) || L == 0 || L > 16) return -1;
    for (uint32_t l = 0; l < L; ++l) {
        const level_t lv = level_of(offsets, l, S, H, scales);
        for (uint32_t b = 0; b < B; ++b) {
            uint32_t pg[3], pl[3];
            float pos[3], deriv[3];
            if (!cell_of(D, inputs + (size_t)b * D, &lv, align, interp, pg, pos, deriv)) continue;
            const float *g = grad + ((size_t)l * B + b) * 2;
            for (uint32_t idx = 0; idx < (1u << D); ++idx) {
                const float w = corner(D, idx, pg, pos, pl);
                const size_t e = lv.off + (size_t)slot_of(D, gridtype, align, &lv, pl);
                const float t0 = R(w * g[0], rnd), t1 = R(w * g[1], rnd);
                sum[2 * e] += t0;
                sum[2 * e + 1] += t1;
                abs_sum[2 * e] += fabs(t0);
                abs_sum[2 * e + 1] += fabs(t1);
                count[e] += 1;
            }
        }
    }
    return 0;
}

/* input gradient: grad [L,B,2], dy_dx [B,L,D,2] -> grad_inputs [B,D] */
int ghc_input_grad(const float *grad, const float *dy_dx, uint32_t B, uint32_t D, uint32_t L, int rnd, float *grad_inputs) {
    for (uint32_t b = 0; b < B; ++b)
        for (uint32_t d = 0; d < D; ++d) {
            float r = 0.f;
            for (uint32_t l = 0; l < L; ++l)
                for (uint32_t ch = 0; ch < 2; ++ch)
                    r = R(r + R(grad[((size_t)l * B + b) * 2 + ch] * dy_dx[(((size_t)b * L + l) * D + d) * 2 + ch], rnd), rnd);
            grad_inputs[(size_t)b * D + d] = r;
        }
    return 0;
}
