/*
 * tvl1_gpu_model.c -- C/OpenMP restatement of oracle/tvl1_gpu_model.py (the CUDA semantics of the reference's
 * cv::cuda::OpticalFlowDual_TVL1), operation for operation, so that the engine can be checked against it at
 * full frame sizes (the numpy model needs minutes there).
 *
 * TEST INFRASTRUCTURE -- never linked into libb200flow.so.
 *
 * One source, three builds (oracle/Makefile):
 *   REAL = float   _build/libtvl1_gpu_model_f32.so   the reference's CUDA semantics in float; equals the numpy model
 *                  bit for bit (tests/test_oracle_cpu.py) -- every float operation is one rounded IEEE operation in
 *                  the numpy model's order, -ffp-contract=off keeps the compiler from fusing any of them;
 *   REAL = double  _build/libtvl1_gpu_model_f64.so   the same algorithm in double: the yardstick for how far float
 *                  rounding alone moves the flow;
 *   REAL = float, ENGINE_ROUNDING   _build/libtvl1_gpu_model_eng.so   the engine's own roundings, which the engine must
 *                  equal bit for bit.  It departs from the f32 build exactly where the engine does (DESIGN.md §4.1):
 *                    - the thresholding divides by multiplying with rcp.approx(|grad I|^2), stored once per warp
 *                      (tvl1_inv_grad: 1e30 where |grad I|^2 <= FLT_EPSILON), and the three-way test is a clamp;
 *                    - |grad u| is sqrt.approx(fma(ux, ux, uy * uy)); the dual update of (u1, u2) divides through one
 *                      shared rcp.approx(a1 * a2), that of u3 (gamma) through rcp.approx(a);
 *                    - the divergence takes a zero ghost on the first row / column: (p - 0) + (q - q_up);
 *                    - the warp uses the Keys weights expanded in t and contracted as nvcc contracts them
 *                      (keys_weights in csrc/tvl1.cu), separable sums for interior pixels and tap-by-tap clamped sums
 *                      where the 6 x 6 window touches the image border, classified as k_tvl1_warp_sep does;
 *                    - fmaf() wherever the kernels fuse (the bilinear resize taps included);
 *                    - an optional median pass (the engine's MEDIAN_FILTERING / MEDIAN_PERIOD knobs).
 *                  rcp.approx.ftz / sqrt.approx.ftz are emulated from tables of their device values over [1, 2) and
 *                  [1, 4) with the exponent scaled and the .ftz rules applied (tvl1_model_set_mufu_tables); the
 *                  emulation is checked against the device on all 2^32 inputs (tests/test_tvl1_gpu.py).
 * Constants that are part of the algorithm (the float32 epsilon of the thresholding step) keep their value in all.
 * The median pass (medianFiltering 3 or 5) is exact selection, so every build applies it the same way.
 *
 * Parallelism: `omp parallel for` over rows in every per-pixel stage; each pixel's result depends on the inputs
 * only, never on the thread count.  The error image is summed in double by numpy's pairwise summation (blocks of
 * 128, eight accumulators), serially, so the epsilon cadence decides exactly as the numpy model does.
 */
#include <float.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifndef REAL
#define REAL float
#endif
typedef REAL real;
#define IS_DOUBLE (sizeof(real) == sizeof(double))

static real r_floor(real v) { return IS_DOUBLE ? (real)floor((double)v) : (real)floorf((float)v); }
static real r_ceil(real v) { return IS_DOUBLE ? (real)ceil((double)v) : (real)ceilf((float)v); }
static real r_abs(real v) { return IS_DOUBLE ? (real)fabs((double)v) : (real)fabsf((float)v); }
/* numpy's float32 hypot is libm's hypotf, its float64 hypot libm's hypot */
static real r_hypot(real a, real b) { return IS_DOUBLE ? (real)hypot((double)a, (double)b) : (real)hypotf((float)a, (float)b); }

typedef struct {
    double tau, lambda, theta;
    int nscales, warps;
    double epsilon;
    int iterations;
    double scaleStep, gamma;
    int useInitialFlow;
    int medianFiltering; /* 1 off, 3 or 5: cv::medianBlur of (u1, u2) every medianPeriod inner iterations */
    int medianPeriod;    /* 0: once per warp */
} tvl1_model_params;

/* what the caller wants back besides the flow (any pointer may be NULL) */
typedef struct {
    int *iters;          /* per solved level (coarsest first) and warp: inner iterations run */
    int iters_cap;
    int n_iters;
    double *ratios;      /* every sampled error sum divided by its level's scaledEpsilon, in order */
    int ratios_cap;
    int n_ratios;
} tvl1_model_trace;

static int cv_round(double v) { return (int)rint(v); } /* np.rint: round half to even */

static real *alloc_plane(size_t n) { return (real *)calloc(n ? n : 1, sizeof(real)); }

int tvl1_model_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
#else
    (void)n;
    return 1;
#endif
}

int tvl1_model_real_bytes(void) { return (int)sizeof(real); }

#ifdef ENGINE_ROUNDING
int tvl1_model_engine_rounding(void) { return 1; }

/* ---- rcp.approx.ftz.f32 / sqrt.approx.ftz.f32 from tables of their values on [1, 2) and [1, 4) ---- */
static float *rcp_tab;  /* 2^23: rcp.approx of the float with bits 0x3f800000 + m */
static float *sqrt_tab; /* 2^24: sqrt.approx of the float with bits 0x3f800000 + i, i = (exponent parity << 23) | m */

static uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

/* rcp: NaN -> NaN, +-inf -> +-0, +-0 and denormals (.ftz) -> +-inf; otherwise the table value of the mantissa with its
 * exponent lowered by the input's, flushed to +-0 below FLT_MIN */
float tvl1_model_rcp_approx(float x) {
    const uint32_t b = f2u(x), s = b & 0x80000000u, e = (b >> 23) & 0xffu, m = b & 0x7fffffu;
    if (e == 0xffu) return m ? x : u2f(s);
    if (e == 0) return u2f(s | 0x7f800000u);
    const uint32_t y = f2u(rcp_tab[m]);
    const int ef = (int)((y >> 23) & 0xffu) - ((int)e - 127);
    return ef <= 0 ? u2f(s) : u2f(s | ((uint32_t)ef << 23) | (y & 0x7fffffu));
}

/* sqrt: +-0 and denormals (.ftz) -> +-0, other negatives -> NaN, +inf -> +inf, NaN -> NaN; otherwise the table value of
 * the mantissa and exponent parity with half the remaining (even) exponent added */
float tvl1_model_sqrt_approx(float x) {
    const uint32_t b = f2u(x), s = b & 0x80000000u, e = (b >> 23) & 0xffu, m = b & 0x7fffffu;
    if (e == 0) return u2f(s);
    if (s) return NAN;
    if (e == 0xffu) return x;
    const int E = (int)e - 127, par = E & 1;
    const uint32_t y = f2u(sqrt_tab[((uint32_t)par << 23) | m]);
    const int ef = (int)((y >> 23) & 0xffu) + (E - par) / 2;
    return u2f(((uint32_t)ef << 23) | (y & 0x7fffffu));
}

/* the tables, copied; returns 0 */
int tvl1_model_set_mufu_tables(const float *rcp, const float *sq) {
    float *a = (float *)malloc(sizeof(float) << 23), *b = (float *)malloc(sizeof(float) << 24);
    if (!a || !b) {
        free(a); free(b);
        return -1;
    }
    memcpy(a, rcp, sizeof(float) << 23);
    memcpy(b, sq, sizeof(float) << 24);
    free(rcp_tab); free(sqrt_tab);
    rcp_tab = a;
    sqrt_tab = b;
    return 0;
}

/* out[i] = op(in[i]), op 0 rcp, 1 sqrt: the emulation in bulk, for the tests */
int tvl1_model_mufu_apply(int op, const float *in, float *out, long n) {
    if (!rcp_tab || !sqrt_tab) return -3;
#pragma omp parallel for schedule(static)
    for (long i = 0; i < n; i++) out[i] = op == 0 ? tvl1_model_rcp_approx(in[i]) : tvl1_model_sqrt_approx(in[i]);
    return 0;
}
#else
int tvl1_model_engine_rounding(void) { return 0; }
#endif

/* numpy's pairwise_sum (numpy/_core/src/umath/loops_utils.h.src) for a contiguous array, as np.sum calls it */
static double pairwise_sum(const real *a, long n) {
    if (n < 8) {
        double res = 0.;
        for (long i = 0; i < n; i++) res += (double)a[i];
        return res;
    } else if (n <= 128) {
        double r[8], res;
        long i;
        for (int k = 0; k < 8; k++) r[k] = (double)a[k];
        for (i = 8; i < n - (n % 8); i += 8)
            for (int k = 0; k < 8; k++) r[k] += (double)a[i + k];
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; i++) res += (double)a[i];
        return res;
    } else {
        long n2 = n / 2;
        n2 -= n2 % 8;
        return pairwise_sum(a, n2) + pairwise_sum(a + n2, n - n2);
    }
}

double tvl1_model_sum(const real *a, long n) { return 0. + pairwise_sum(a, n); }

/* cv::cuda::resize INTER_LINEAR (model: resize_linear): src = dst * float(1/f), right / bottom taps clamped */
static void resize_linear(const real *src, int H, int W, real *dst, int dh, int dw, double fx, double fy) {
    if (dh == H && dw == W) {
        memcpy(dst, src, sizeof(real) * (size_t)H * W);
        return;
    }
    const real sx = (real)(1.0 / fx), sy = (real)(1.0 / fy);
#pragma omp parallel for schedule(static)
    for (int y = 0; y < dh; y++) {
        const real src_y = (real)y * sy;
        const long y1 = (long)r_floor(src_y), y2 = y1 + 1;
        const long y1c = y1 < H - 1 ? y1 : H - 1, y2r = y2 < H - 1 ? y2 : H - 1;
        const real wy2 = (real)y2 - src_y, wy1 = src_y - (real)y1;
        for (int x = 0; x < dw; x++) {
            const real src_x = (real)x * sx;
            const long x1 = (long)r_floor(src_x), x2 = x1 + 1;
            const long x1c = x1 < W - 1 ? x1 : W - 1, x2r = x2 < W - 1 ? x2 : W - 1;
            const real wx2 = (real)x2 - src_x, wx1 = src_x - (real)x1;
            real out = 0;
#ifdef ENGINE_ROUNDING /* resize_sample in csrc/pyramid.cu: one fma per tap */
            out = fmaf(src[y1c * W + x1c], wx2 * wy2, out);
            out = fmaf(src[y1c * W + x2r], wx1 * wy2, out);
            out = fmaf(src[y2r * W + x1c], wx2 * wy1, out);
            out = fmaf(src[y2r * W + x2r], wx1 * wy1, out);
#else
            out = out + src[y1c * W + x1c] * (wx2 * wy2);
            out = out + src[y1c * W + x2r] * (wx1 * wy2);
            out = out + src[y2r * W + x1c] * (wx2 * wy1);
            out = out + src[y2r * W + x2r] * (wx1 * wy1);
#endif
            dst[(size_t)y * dw + x] = out;
        }
    }
}

static void scale_plane(real *a, size_t n, real f) {
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) a[i] = a[i] * f;
}

static long clampl(long v, long lo, long hi) { return v < lo ? lo : (v > hi ? hi : v); }

#ifndef ENGINE_ROUNDING /* the reference's expressions, one IEEE operation each (the f32 and f64 builds) */
/* centeredGradientKernel: clamped central difference * 0.5 */
static void centered_gradient(const real *src, int H, int W, real *dx, real *dy) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        const int yp = y + 1 < H - 1 ? y + 1 : H - 1, ym = y - 1 > 0 ? y - 1 : 0;
        for (int x = 0; x < W; x++) {
            const int xp = x + 1 < W - 1 ? x + 1 : W - 1, xm = x - 1 > 0 ? x - 1 : 0;
            dx[(size_t)y * W + x] = (real)0.5 * (src[(size_t)y * W + xp] - src[(size_t)y * W + xm]);
            dy[(size_t)y * W + x] = (real)0.5 * (src[(size_t)yp * W + x] - src[(size_t)ym * W + x]);
        }
    }
}

/* bicubicCoeff: Keys kernel, a = -0.5 */
static real bicubic_coeff(real x) {
    x = r_abs(x);
    if (x <= 1) return x * x * ((real)1.5 * x - (real)2.5) + (real)1.0;
    if (x < 2) return x * (x * ((real)-0.5 * x + (real)2.5) - (real)4.0) + (real)2.0;
    return 0;
}

/* warpBackwardKernel: taps cx in [ceil(wx-2), floor(wx+2)], clamp addressing, weights normalised by their sum.  The
 * numpy model visits a fixed 5 x 5 tap grid and zeroes the weights outside the window; so does this loop. */
static void warp_backward(const real *I0, const real *I1, const real *I1x, const real *I1y, const real *u1,
                          const real *u2, int H, int W, real *I1wx, real *I1wy, real *grad, real *rho) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            const size_t i = (size_t)y * W + x;
            const real wx = (real)x + u1[i], wy = (real)y + u2[i];
            const long xmin = (long)r_ceil(wx - (real)2.0), xmax = (long)r_floor(wx + (real)2.0);
            const long ymin = (long)r_ceil(wy - (real)2.0), ymax = (long)r_floor(wy + (real)2.0);
            real s = 0, sx = 0, sy = 0, ws = 0;
            for (int j = 0; j < 5; j++) {
                const long cy = ymin + j;
                const int my = cy <= ymax;
                const long cyc = clampl(cy, 0, H - 1);
                const real ky = bicubic_coeff(wy - (real)cy);
                for (int t = 0; t < 5; t++) {
                    const long cx = xmin + t;
                    const int m = my && cx <= xmax;
                    const long cxc = clampl(cx, 0, W - 1);
                    const real wgt = m ? bicubic_coeff(wx - (real)cx) * ky : (real)0;
                    const size_t k = (size_t)cyc * W + cxc;
                    s = s + wgt * I1[k];
                    sx = sx + wgt * I1x[k];
                    sy = sy + wgt * I1y[k];
                    ws = ws + wgt;
                }
            }
            const real coeff = (real)1.0 / ws;
            const real w1 = s * coeff, wgx = sx * coeff, wgy = sy * coeff;
            I1wx[i] = wgx;
            I1wy[i] = wgy;
            grad[i] = wgx * wgx + wgy * wgy;
            rho[i] = w1 - wgx * u1[i] - wgy * u2[i] - I0[i];
        }
    }
}

/* divergence of (v1, v2) at (y, x), backward differences, first row / column as in the reference */
static real divergence_at(const real *v1, const real *v2, int W, int y, int x) {
    const size_t i = (size_t)y * W + x;
    if (y > 0 && x > 0) return (v1[i] - v1[i - 1]) + (v2[i] - v2[i - W]);
    if (y > 0) return v1[i] + v2[i] - v2[i - W];
    if (x > 0) return v1[i] - v1[i - 1] + v2[i];
    return v1[i] + v2[i];
}

/* estimateUKernel, in place: each pixel reads and writes only its own u, the p planes are read-only here */
static void estimate_u(const real *I1wx, const real *I1wy, const real *grad, const real *rho_c, const real *p11,
                       const real *p12, const real *p21, const real *p22, const real *p31, const real *p32, real *u1,
                       real *u2, real *u3, int H, int W, real l_t, real theta, real gamma, int use_gamma, real *err) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            const size_t i = (size_t)y * W + x;
            const real Ix = I1wx[i], Iy = I1wy[i], g = grad[i];
            const real u1o = u1[i], u2o = u2[i];
            const real u3o = use_gamma ? u3[i] : (real)0;
            const real rho = rho_c[i] + (Ix * u1o + Iy * u2o + gamma * u3o);
            const int c1 = rho < -l_t * g;
            const int c2 = !c1 && rho > l_t * g;
            const int c3 = !c1 && !c2 && g > (real)FLT_EPSILON;
            const real fi = c3 ? -rho / g : (real)0;
#define SEL(a) (c1 ? l_t * (a) : (c2 ? -l_t * (a) : (c3 ? fi * (a) : (real)0)))
            const real v1 = u1o + SEL(Ix);
            const real v2 = u2o + SEL(Iy);
            const real n1 = v1 + theta * divergence_at(p11, p12, W, y, x);
            const real n2 = v2 + theta * divergence_at(p21, p22, W, y, x);
            if (use_gamma) {
                const real v3 = u3o + SEL(gamma);
                u3[i] = v3 + theta * divergence_at(p31, p32, W, y, x);
            }
#undef SEL
            u1[i] = n1;
            u2[i] = n2;
            err[i] = (u1o - n1) * (u1o - n1) + (u2o - n2) * (u2o - n2); /* u3 is not part of the GPU error */
        }
    }
}

/* estimateDualVariablesKernel for one (u, pa, pb) triple, in place: forward differences, zero on the last row /
 * column, p = (p + taut * grad u) / (1 + taut * |grad u|) */
static void estimate_dual_one(const real *u, real *pa, real *pb, int H, int W, real taut) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            const size_t i = (size_t)y * W + x;
            const real ux = x < W - 1 ? u[i + 1] - u[i] : (real)0;
            const real uy = y < H - 1 ? u[i + W] - u[i] : (real)0;
            const real g = r_hypot(ux, uy);
            const real ng = (real)1.0 + taut * g;
            pa[i] = (pa[i] + taut * ux) / ng;
            pb[i] = (pb[i] + taut * uy) / ng;
        }
    }
}
#endif /* !ENGINE_ROUNDING */

#ifdef ENGINE_ROUNDING
/* ---- the engine's roundings (csrc/tvl1.cu, csrc/tvl1_math.cuh); float only ---- */

/* keys_weights as nvcc contracts it (see its comment in csrc/tvl1.cu) */
static void keys_weights(float t, float k[4]) {
    k[0] = fmaf(fmaf(-0.5f, t, 1.0f), t, -0.5f) * t;
    k[1] = fmaf(fmaf(1.5f, t, -2.5f) * t, t, 1.0f);
    k[2] = fmaf(fmaf(-1.5f, t, 2.0f), t, 0.5f) * t;
    k[3] = (fmaf(0.5f, t, -0.5f) * t) * t;
}

static float tvl1_inv_grad(float g) { return g > FLT_EPSILON ? tvl1_model_rcp_approx(g) : 1e30f; }

/* k_tvl1_warp_sep (the tiled kernel is bit-identical to it): the gradient of I1 is formed at the taps, the grad plane
 * receives tvl1_inv_grad(|grad I1w|^2) */
static void warp_backward(const float *I0, const float *I1, const float *u1, const float *u2, int H, int W,
                          float *I1wx, float *I1wy, float *grad, float *rho) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            const size_t i = (size_t)y * W + x;
            const float wx = (float)x + u1[i], wy = (float)y + u2[i];
            const float fx = floorf(wx), fy = floorf(wy);
            const int ix = (int)fminf(fmaxf(fx, -8.f), (float)W + 8.f) - 1;
            const int iy = (int)fminf(fmaxf(fy, -8.f), (float)H + 8.f) - 1;
            float kx[4], ky[4], sum, sumx, sumy;
            keys_weights(wx - fx, kx);
            keys_weights(wy - fy, ky);
            const float wsum = ((kx[0] + kx[1]) + (kx[2] + kx[3])) * ((ky[0] + ky[1]) + (ky[2] + ky[3]));
            if (ix >= 1 && iy >= 1 && ix + 4 <= W - 1 && iy + 4 <= H - 1) { /* separable: rows iy-1.., columns ix-1.. */
                float r[6], rx[4];
                for (int j = 0; j < 6; j++) {
                    const float *a = I1 + (size_t)(iy - 1 + j) * W + (ix - 1);
                    r[j] = fmaf(kx[3], a[4], fmaf(kx[2], a[3], fmaf(kx[1], a[2], kx[0] * a[1])));
                    if (j >= 1 && j <= 4)
                        rx[j - 1] = fmaf(kx[3], a[5] - a[3], fmaf(kx[2], a[4] - a[2], fmaf(kx[1], a[3] - a[1], kx[0] * (a[2] - a[0]))));
                }
                sum = fmaf(ky[3], r[4], fmaf(ky[2], r[3], fmaf(ky[1], r[2], ky[0] * r[1])));
                sumx = 0.5f * fmaf(ky[3], rx[3], fmaf(ky[2], rx[2], fmaf(ky[1], rx[1], ky[0] * rx[0])));
                sumy = 0.5f * fmaf(ky[3], r[5] - r[3], fmaf(ky[2], r[4] - r[2], fmaf(ky[1], r[3] - r[1], ky[0] * (r[2] - r[0]))));
            } else { /* warp_border_taps: clamped taps, clamped-neighbour gradients */
                sum = sumx = sumy = 0.f;
                for (int j = 0; j < 4; j++) {
                    const long cy = clampl(iy + j, 0, H - 1), cyp = cy + 1 < H - 1 ? cy + 1 : H - 1, cym = cy - 1 > 0 ? cy - 1 : 0;
                    for (int t = 0; t < 4; t++) {
                        const long cx = clampl(ix + t, 0, W - 1), cxp = cx + 1 < W - 1 ? cx + 1 : W - 1, cxm = cx - 1 > 0 ? cx - 1 : 0;
                        const float w = kx[t] * ky[j];
                        const float gx = 0.5f * (I1[cy * W + cxp] - I1[cy * W + cxm]);
                        const float gy = 0.5f * (I1[cyp * W + cx] - I1[cym * W + cx]);
                        sum = fmaf(w, I1[cy * W + cx], sum);
                        sumx = fmaf(w, gx, sumx);
                        sumy = fmaf(w, gy, sumy);
                    }
                }
            }
            const float coeff = 1.0f / wsum;
            const float I1w = sum * coeff, Ix = sumx * coeff, Iy = sumy * coeff;
            I1wx[i] = Ix;
            I1wy[i] = Iy;
            grad[i] = tvl1_inv_grad(fmaf(Iy, Iy, Ix * Ix));
            rho[i] = fmaf(-Iy, u2[i], fmaf(-Ix, u1[i], I1w)) - I0[i];
        }
    }
}

/* tvl1_threshold: the clamp of -rho / |grad|^2, with the stored reciprocal */
static float tvl1_threshold(float rho, float inv_grad, float l_t) { return fminf(fmaxf(-rho * inv_grad, -l_t), l_t); }

/* divergence with the zero ghost on the first row / column */
static float divergence_ghost(const float *a, const float *b, int W, int y, int x) {
    const size_t i = (size_t)y * W + x;
    return (a[i] - (x > 0 ? a[i - 1] : 0.f)) + (b[i] - (y > 0 ? b[i - W] : 0.f));
}

/* k_tvl1_estimate_u (tvl1_update_u when gamma == 0), in place */
static void estimate_u(const float *I1wx, const float *I1wy, const float *grad, const float *rho_c, const float *p11,
                       const float *p12, const float *p21, const float *p22, const float *p31, const float *p32, float *u1,
                       float *u2, float *u3, int H, int W, float l_t, float theta, float gamma, int use_gamma, float *err) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            const size_t i = (size_t)y * W + x;
            const float Ix = I1wx[i], Iy = I1wy[i], ig = grad[i];
            const float u1o = u1[i], u2o = u2[i];
            float rho;
            if (use_gamma) rho = rho_c[i] + fmaf(gamma, u3[i], fmaf(Iy, u2o, Ix * u1o));
            else rho = fmaf(Iy, u2o, fmaf(Ix, u1o, rho_c[i]));
            const float fi = tvl1_threshold(rho, ig, l_t);
            const float n1 = fmaf(theta, divergence_ghost(p11, p12, W, y, x), fmaf(fi, Ix, u1o));
            const float n2 = fmaf(theta, divergence_ghost(p21, p22, W, y, x), fmaf(fi, Iy, u2o));
            if (use_gamma) u3[i] = fmaf(theta, divergence_ghost(p31, p32, W, y, x), fmaf(fi, gamma, u3[i]));
            u1[i] = n1;
            u2[i] = n2;
            const float d1 = u1o - n1, d2 = u2o - n2;
            err[i] = fmaf(d2, d2, d1 * d1);
        }
    }
}

/* forward differences of u at (y, x), zero on the last column / row */
static void fwd_diff(const float *u, int H, int W, int y, int x, float *ux, float *uy) {
    const size_t i = (size_t)y * W + x;
    *ux = x < W - 1 ? u[i + 1] - u[i] : 0.f;
    *uy = y < H - 1 ? u[i + W] - u[i] : 0.f;
}

/* k_tvl1_estimate_dual: tvl1_update_p2 for (u1, u2), tvl1_update_p for u3; in place */
static void estimate_dual(const float *u1, const float *u2, const float *u3, float *p11, float *p12, float *p21,
                          float *p22, float *p31, float *p32, int H, int W, float taut, int use_gamma) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            const size_t i = (size_t)y * W + x;
            float ux1, uy1, ux2, uy2;
            fwd_diff(u1, H, W, y, x, &ux1, &uy1);
            fwd_diff(u2, H, W, y, x, &ux2, &uy2);
            const float g1 = tvl1_model_sqrt_approx(fmaf(ux1, ux1, uy1 * uy1));
            const float g2 = tvl1_model_sqrt_approx(fmaf(ux2, ux2, uy2 * uy2));
            const float a1 = fmaf(taut, g1, 1.0f), a2 = fmaf(taut, g2, 1.0f);
            const float r = tvl1_model_rcp_approx(a1 * a2);
            const float inv1 = r * a2, inv2 = r * a1;
            p11[i] = fmaf(taut, ux1, p11[i]) * inv1;
            p12[i] = fmaf(taut, uy1, p12[i]) * inv1;
            p21[i] = fmaf(taut, ux2, p21[i]) * inv2;
            p22[i] = fmaf(taut, uy2, p22[i]) * inv2;
            if (use_gamma) {
                float ux, uy;
                fwd_diff(u3, H, W, y, x, &ux, &uy);
                const float g = tvl1_model_sqrt_approx(fmaf(ux, ux, uy * uy));
                const float inv = tvl1_model_rcp_approx(fmaf(taut, g, 1.0f));
                p31[i] = fmaf(taut, ux, p31[i]) * inv;
                p32[i] = fmaf(taut, uy, p32[i]) * inv;
            }
        }
    }
}
#endif /* ENGINE_ROUNDING */

/* cv::medianBlur of one plane, ksize 3 or 5, replicated border (k_tvl1_median): src -> dst */
static void median_plane(const real *src, real *dst, int H, int W, int ks) {
    const int R = ks / 2, N = ks * ks;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; y++) {
        for (int x = 0; x < W; x++) {
            real w[25];
            for (int j = 0; j < ks; j++)
                for (int i = 0; i < ks; i++)
                    w[j * ks + i] = src[clampl(y + j - R, 0, H - 1) * W + clampl(x + i - R, 0, W - 1)];
            for (int a = 1; a < N; a++) { /* insertion sort; the middle element is the median */
                const real v = w[a];
                int b = a - 1;
                for (; b >= 0 && w[b] > v; b--) w[b + 1] = w[b];
                w[b + 1] = v;
            }
            dst[(size_t)y * W + x] = w[N / 2];
        }
    }
}

static void trace_iters(tvl1_model_trace *tr, int n) {
    if (tr && tr->iters && tr->n_iters < tr->iters_cap) tr->iters[tr->n_iters] = n;
    if (tr) tr->n_iters++;
}
static void trace_ratio(tvl1_model_trace *tr, double r) {
    if (tr && tr->ratios && tr->n_ratios < tr->ratios_cap) tr->ratios[tr->n_ratios] = r;
    if (tr) tr->n_ratios++;
}

/* procOneScale incl. the reference's error cadence (model: proc_one_scale).  Returns 0, or -1 out of memory. */
static int proc_one_scale(const tvl1_model_params *P, const real *I0, const real *I1, int h, int w, real *u1, real *u2,
                          real *u3, tvl1_model_trace *tr) {
    const size_t n = (size_t)h * w;
    const double scaledEpsilon = P->epsilon * P->epsilon * (double)n;
    const int use_gamma = P->gamma != 0;
    const int med_k = (P->medianFiltering == 3 || P->medianFiltering == 5) ? P->medianFiltering : 1;
    const int med_period = P->medianPeriod > 0 ? P->medianPeriod : (P->iterations > 0 ? P->iterations : 1);
    const int nbuf = med_k > 1 ? 15 : 13;
    real *buf[15];
    for (int i = 0; i < 15; i++) buf[i] = NULL;
    int ok = 1;
    for (int i = 0; i < nbuf && ok; i++) ok = (buf[i] = alloc_plane(n)) != NULL;
    int rc = -1;
    if (!ok) goto done;
    real *I1x = buf[0], *I1y = buf[1], *I1wx = buf[2], *I1wy = buf[3], *grad = buf[4], *rho_c = buf[5];
    real *p11 = buf[6], *p12 = buf[7], *p21 = buf[8], *p22 = buf[9], *p31 = buf[10], *p32 = buf[11], *err = buf[12];
    real *med1 = buf[13], *med2 = buf[14]; /* the median pass's output, copied back (medianFiltering 3 / 5 only) */
    const real l_t = (real)(P->lambda * P->theta);
    const real taut = (real)(P->tau / P->theta);
    const real theta = (real)P->theta, gamma = (real)P->gamma;
#ifdef ENGINE_ROUNDING
    (void)I1x; (void)I1y;
#else
    centered_gradient(I1, h, w, I1x, I1y);
#endif
    for (int wi = 0; wi < P->warps; wi++) {
#ifdef ENGINE_ROUNDING
        warp_backward(I0, I1, u1, u2, h, w, I1wx, I1wy, grad, rho_c);
#else
        warp_backward(I0, I1, I1x, I1y, u1, u2, h, w, I1wx, I1wy, grad, rho_c);
#endif
        double error = DBL_MAX, prevError = 0.0;
        int it = 0;
        while (error > scaledEpsilon && it < P->iterations) {
            if (med_k > 1 && it % med_period == 0) { /* the engine's outer loop: median, then `period` iterations */
                median_plane(u1, med1, h, w, med_k);
                median_plane(u2, med2, h, w, med_k);
                memcpy(u1, med1, sizeof(real) * n);
                memcpy(u2, med2, sizeof(real) * n);
            }
            const int calcError = (P->epsilon > 0) && (it & 1) && (prevError < scaledEpsilon);
            estimate_u(I1wx, I1wy, grad, rho_c, p11, p12, p21, p22, p31, p32, u1, u2, u3, h, w, l_t, theta, gamma,
                       use_gamma, err);
            if (calcError) {
                error = tvl1_model_sum(err, (long)n);
                prevError = error;
                trace_ratio(tr, error / scaledEpsilon);
            } else {
                error = DBL_MAX;
                prevError -= scaledEpsilon;
            }
#ifdef ENGINE_ROUNDING
            estimate_dual(u1, u2, u3, p11, p12, p21, p22, p31, p32, h, w, taut, use_gamma);
#else
            estimate_dual_one(u1, p11, p12, h, w, taut);
            estimate_dual_one(u2, p21, p22, h, w, taut);
            if (use_gamma) estimate_dual_one(u3, p31, p32, h, w, taut);
#endif
            it++;
        }
        trace_iters(tr, it);
    }
    rc = 0;
done:
    for (int i = 0; i < 15; i++) free(buf[i]);
    return rc;
}

/* OpticalFlowDual_TVL1_Impl::calc (model: calc).  I0, I1: h x w, already converted to float (u8 values exact);
 * is_u8 selects the convertTo factor (1 for 8-bit input, 255 for float input).  init_flow: h x w x 2 or NULL.
 * flow: h x w x 2 of `real`.  Returns 0, -1 out of memory, -2 bad parameters. */
int tvl1_model_calc(const tvl1_model_params *P, const float *I0, const float *I1, int h, int w, int is_u8,
                    const float *init_flow, real *flow, tvl1_model_trace *tr) {
    if (!P || P->nscales <= 0 || h <= 0 || w <= 0 || (P->useInitialFlow && !init_flow)) return -2;
#ifdef ENGINE_ROUNDING
    if (!rcp_tab || !sqrt_tab) return -3;
#endif
    if (tr) tr->n_iters = tr->n_ratios = 0;
    const int ns_param = P->nscales;
    int *hs = (int *)calloc((size_t)ns_param, sizeof(int)), *ws = (int *)calloc((size_t)ns_param, sizeof(int));
    real **I0s = (real **)calloc((size_t)ns_param, sizeof(real *)), **I1s = (real **)calloc((size_t)ns_param, sizeof(real *));
    real **u1s = (real **)calloc((size_t)ns_param, sizeof(real *)), **u2s = (real **)calloc((size_t)ns_param, sizeof(real *));
    real *u3 = NULL, *u3n = NULL;
    int rc = -1, nscales = ns_param;
    if (!hs || !ws || !I0s || !I1s || !u1s || !u2s) goto done;
    const real k = is_u8 ? (real)1.0 : (real)255.0;
    const size_t n0 = (size_t)h * w;
    hs[0] = h;
    ws[0] = w;
    if (!(I0s[0] = alloc_plane(n0)) || !(I1s[0] = alloc_plane(n0)) || !(u1s[0] = alloc_plane(n0)) ||
        !(u2s[0] = alloc_plane(n0)))
        goto done;
    for (size_t i = 0; i < n0; i++) {
        I0s[0][i] = (real)I0[i] * k;
        I1s[0][i] = (real)I1[i] * k;
        if (P->useInitialFlow) {
            u1s[0][i] = (real)init_flow[2 * i];
            u2s[0][i] = (real)init_flow[2 * i + 1];
        }
    }
    for (int s = 1; s < ns_param; s++) {
        const int ph = hs[s - 1], pw = ws[s - 1];
        const int nh = cv_round(ph * P->scaleStep), nw = cv_round(pw * P->scaleStep);
        const size_t nn = (size_t)nh * nw;
        hs[s] = nh;
        ws[s] = nw;
        if (!(I0s[s] = alloc_plane(nn)) || !(I1s[s] = alloc_plane(nn))) goto done;
        resize_linear(I0s[s - 1], ph, pw, I0s[s], nh, nw, P->scaleStep, P->scaleStep);
        resize_linear(I1s[s - 1], ph, pw, I1s[s], nh, nw, P->scaleStep, P->scaleStep);
        if (nw < 16 || nh < 16) { /* built, not used (< 16 px early stop) */
            nscales = s;
            break;
        }
        if (!(u1s[s] = alloc_plane(nn)) || !(u2s[s] = alloc_plane(nn))) goto done;
        if (P->useInitialFlow) {
            resize_linear(u1s[s - 1], ph, pw, u1s[s], nh, nw, P->scaleStep, P->scaleStep);
            resize_linear(u2s[s - 1], ph, pw, u2s[s], nh, nw, P->scaleStep, P->scaleStep);
            scale_plane(u1s[s], nn, (real)P->scaleStep);
            scale_plane(u2s[s], nn, (real)P->scaleStep);
        }
    }
    const int use_gamma = P->gamma != 0;
    if (use_gamma) {
        if (!(u3 = alloc_plane(n0)) || !(u3n = alloc_plane(n0))) goto done; /* zero at the coarsest level */
    }
    for (int s = nscales - 1; s >= 0; s--) {
        if (proc_one_scale(P, I0s[s], I1s[s], hs[s], ws[s], u1s[s], u2s[s], u3, tr)) goto done;
        if (s == 0) break;
        const int dh = hs[s - 1], dw = ws[s - 1];
        const double fx = (double)dw / ws[s], fy = (double)dh / hs[s];
        const real inv = (real)(1.0 / P->scaleStep);
        resize_linear(u1s[s], hs[s], ws[s], u1s[s - 1], dh, dw, fx, fy);
        resize_linear(u2s[s], hs[s], ws[s], u2s[s - 1], dh, dw, fx, fy);
        scale_plane(u1s[s - 1], (size_t)dh * dw, inv);
        scale_plane(u2s[s - 1], (size_t)dh * dw, inv);
        if (use_gamma) { /* resized, not rescaled */
            resize_linear(u3, hs[s], ws[s], u3n, dh, dw, fx, fy);
            real *t = u3;
            u3 = u3n;
            u3n = t;
        }
    }
    for (size_t i = 0; i < n0; i++) {
        flow[2 * i] = u1s[0][i];
        flow[2 * i + 1] = u2s[0][i];
    }
    rc = 0;
done:
    for (int s = 0; s < ns_param; s++) {
        if (I0s) free(I0s[s]);
        if (I1s) free(I1s[s]);
        if (u1s) free(u1s[s]);
        if (u2s) free(u2s[s]);
    }
    free(hs); free(ws); free(I0s); free(I1s); free(u1s); free(u2s); free(u3); free(u3n);
    return rc;
}
