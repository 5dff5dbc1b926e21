/*
 * tvl1_gpu_model.c -- C/OpenMP restatement of oracle/tvl1_gpu_model.py (the CUDA semantics of the reference's
 * cv::cuda::OpticalFlowDual_TVL1), operation for operation, so that the engine can be checked against it at
 * full frame sizes (the numpy model needs minutes there).
 *
 * TEST INFRASTRUCTURE -- never linked into libb200flow.so.
 *
 * One source, two builds (oracle/Makefile):
 *   REAL = float   _build/libtvl1_gpu_model_f32.so   the model the engine must match; equals the numpy model bit
 *                  for bit (tests/test_oracle_cpu.py) -- every float operation is one rounded IEEE operation in
 *                  the numpy model's order, -ffp-contract=off keeps the compiler from fusing any of them;
 *   REAL = double  _build/libtvl1_gpu_model_f64.so   the same algorithm in double: the yardstick for how far float
 *                  rounding alone moves the flow, which sets the tolerances of the full-size engine tests.
 * Constants that are part of the algorithm (the float32 epsilon of the thresholding step) keep their value in both.
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
            out = out + src[y1c * W + x1c] * (wx2 * wy2);
            out = out + src[y1c * W + x2r] * (wx1 * wy2);
            out = out + src[y2r * W + x1c] * (wx2 * wy1);
            out = out + src[y2r * W + x2r] * (wx1 * wy1);
            dst[(size_t)y * dw + x] = out;
        }
    }
}

static void scale_plane(real *a, size_t n, real f) {
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) a[i] = a[i] * f;
}

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

static long clampl(long v, long lo, long hi) { return v < lo ? lo : (v > hi ? hi : v); }

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
    real *buf[14];
    for (int i = 0; i < 14; i++) buf[i] = NULL;
    int ok = 1;
    for (int i = 0; i < 14 && ok; i++) ok = (buf[i] = alloc_plane(n)) != NULL;
    int rc = -1;
    if (!ok) goto done;
    real *I1x = buf[0], *I1y = buf[1], *I1wx = buf[2], *I1wy = buf[3], *grad = buf[4], *rho_c = buf[5];
    real *p11 = buf[6], *p12 = buf[7], *p21 = buf[8], *p22 = buf[9], *p31 = buf[10], *p32 = buf[11], *err = buf[12];
    centered_gradient(I1, h, w, I1x, I1y);
    const real l_t = (real)(P->lambda * P->theta);
    const real taut = (real)(P->tau / P->theta);
    const real theta = (real)P->theta, gamma = (real)P->gamma;
    for (int wi = 0; wi < P->warps; wi++) {
        warp_backward(I0, I1, I1x, I1y, u1, u2, h, w, I1wx, I1wy, grad, rho_c);
        double error = DBL_MAX, prevError = 0.0;
        int it = 0;
        while (error > scaledEpsilon && it < P->iterations) {
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
            estimate_dual_one(u1, p11, p12, h, w, taut);
            estimate_dual_one(u2, p21, p22, h, w, taut);
            if (use_gamma) estimate_dual_one(u3, p31, p32, h, w, taut);
            it++;
        }
        trace_iters(tr, it);
    }
    rc = 0;
done:
    for (int i = 0; i < 14; i++) free(buf[i]);
    return rc;
}

/* OpticalFlowDual_TVL1_Impl::calc (model: calc).  I0, I1: h x w, already converted to float (u8 values exact);
 * is_u8 selects the convertTo factor (1 for 8-bit input, 255 for float input).  init_flow: h x w x 2 or NULL.
 * flow: h x w x 2 of `real`.  Returns 0, -1 out of memory, -2 bad parameters. */
int tvl1_model_calc(const tvl1_model_params *P, const float *I0, const float *I1, int h, int w, int is_u8,
                    const float *init_flow, real *flow, tvl1_model_trace *tr) {
    if (!P || P->nscales <= 0 || h <= 0 || w <= 0 || (P->useInitialFlow && !init_flow)) return -2;
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
