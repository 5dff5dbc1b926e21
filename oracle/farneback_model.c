/* farneback_model.c -- C/OpenMP restatement of oracle/farneback_gpu_model.calc, in two builds:
 *
 *   f32  (no macro)            restates the numpy float model operation for operation: every float operation
 *                              rounds on its own (-ffp-contract=off), sums in the numpy model's order.  Its flows
 *                              equal calc(precision="f32") bit for bit.
 *   eng  (-DENGINE_ROUNDING)   the roundings of the Farneback engine (opencv_contrib_b200/csrc/farneback.cu,
 *                              pyramid.cu), which the engine must equal bit for bit.
 *
 * Each departure of eng from f32 is one macro (0 / 1), defaulting to ENGINE_ROUNDING, so that it can be switched on
 * alone:
 *   FARN_FMA          the multiply-adds nvcc contracts, as the SASS shows them: a*b + c*d is fmaf(a, b, c*d) (the
 *                     first product fused; updateMatrices' r6*dy + r5*dx is the one exception), a tap chain whose length is known at compile time (polynomial expansion,
 *                     the K = 6 iteration kernels) fuses its centre tap into the first pair, a chain of run-time length
 *                     (level-image blur, generic iteration kernel) starts with a plain product; updateMatrices sums
 *                     r2 + (r4*dy + r6*dx) as the kernel writes it;
 *   FARN_RUNNING_BOX  the box window of the K = 6 kernels (k_farn_iter_fast, k_farn_iter_tma): a balanced tree over
 *                     the first 13 values, then acc + (new - old), restarting at every 16-row strip (origin a multiple
 *                     of 16) and every 4-pixel horizontal task (origin a multiple of 4);
 *   FARN_PYR_TAP5     fastPyramids levels from pyr_tap5 (pyr_tap5.h) instead of the caller's cv2.pyrDown levels;
 *   FARN_FUSED_RESIZE resize_sample of pyramid.cu (one fused multiply-add per tap onto +0) for the level image, the
 *                     flow prolongation and the initial flow;
 *   FARN_SKIP_ZERO    the level image skips bilinear taps whose weight is zero (k_farn_blur_h_resize);
 *   FARN_FLOOR_CLAMP  updateMatrices clamps floorf of the displaced position to [-4, size + 4] before the int
 *                     conversion.  Either way such a pixel has no bilinear cell, so no finite flow changes a bit;
 *                     the clamp keeps the conversion defined.
 *
 * The iteration order argument of farneback_model_calc (0 = fast: the K = 6 kernels, 1 = generic: k_farn_iter) picks
 * the box summation and the first gaussian tap's rounding; it matters only with FARN_RUNNING_BOX / FARN_FMA, and
 * only for winSize 13 (the engine runs every other window size on the generic kernel).
 *
 * Tables (polynomial-expansion constants, level-image and window kernels) come from the caller, so both builds use
 * exactly the values of the model they restate.  TEST INFRASTRUCTURE (see oracle/__init__.py); never linked into
 * libb200flow.so.  Rows are independent within a stage: OpenMP over rows, results do not depend on the thread count. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "pyr_tap5.h"

#ifdef ENGINE_ROUNDING
#define FARN_ENG 1
#else
#define FARN_ENG 0
#endif
#ifndef FARN_FMA
#define FARN_FMA FARN_ENG
#endif
#ifndef FARN_RUNNING_BOX
#define FARN_RUNNING_BOX FARN_ENG
#endif
#ifndef FARN_PYR_TAP5
#define FARN_PYR_TAP5 FARN_ENG
#endif
#ifndef FARN_FUSED_RESIZE
#define FARN_FUSED_RESIZE FARN_ENG
#endif
#ifndef FARN_SKIP_ZERO
#define FARN_SKIP_ZERO FARN_ENG
#endif
#ifndef FARN_FLOOR_CLAMP
#define FARN_FLOOR_CLAMP FARN_ENG
#endif

enum { MIN_SIZE = 32, BORDER_SIZE = 5, USE_INITIAL_FLOW = 4, GAUSSIAN = 256, MAX_LEVELS = 64 };
enum { ORDER_FAST = 0, ORDER_GENERIC = 1 };

int farneback_model_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
#else
    (void)n;
    return 1;
#endif
}

/* which departures this build has: bit 0 FMA, 1 RUNNING_BOX, 2 PYR_TAP5, 3 FUSED_RESIZE, 4 SKIP_ZERO, 5 FLOOR_CLAMP */
int farneback_model_switches(void) {
    return FARN_FMA | FARN_RUNNING_BOX << 1 | FARN_PYR_TAP5 << 2 | FARN_FUSED_RESIZE << 3 | FARN_SKIP_ZERO << 4 |
           FARN_FLOOR_CLAMP << 5;
}

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
static int mini(int a, int b) { return a < b ? a : b; }

/* c + a*b: one fused rounding under FARN_FMA, two otherwise */
static inline float mad(float a, float b, float c) { return FARN_FMA ? fmaf(a, b, c) : c + a * b; }

/* ---- bilinear resize (tvl1_gpu_model.resize_linear / pyramid.cu resize_sample), src = dst * inv, right / bottom taps
 * clamped.  Equal sizes copy.  mul != 1 scales the result (the flow rescale). ---- */
static void resize_linear(const float *src, int sh, int sw, float *dst, int dh, int dw, float mul) {
    if (sh == dh && sw == dw) {
        for (size_t i = 0; i < (size_t)dh * dw; ++i) dst[i] = mul != 1.f ? src[i] * mul : src[i];
        return;
    }
    const float ix = (float)(1.0 / ((double)dw / sw)), iy = (float)(1.0 / ((double)dh / sh));
#pragma omp parallel for schedule(static)
    for (int y = 0; y < dh; ++y) {
        const float sy = (float)y * iy;
        const int y1 = (int)floorf(sy), y2 = y1 + 1;
        const int y1r = mini(y1, sh - 1), y2r = mini(y2, sh - 1);
        const float wy2 = (float)y2 - sy, wy1 = sy - (float)y1;
        for (int x = 0; x < dw; ++x) {
            const float sx = (float)x * ix;
            const int x1 = (int)floorf(sx), x2 = x1 + 1;
            const int x1r = mini(x1, sw - 1), x2r = mini(x2, sw - 1);
            const float wx2 = (float)x2 - sx, wx1 = sx - (float)x1;
            const float *r1 = src + (size_t)y1r * sw, *r2 = src + (size_t)y2r * sw;
            float out = 0.f;
            if (FARN_FUSED_RESIZE) {
                out = fmaf(r1[x1r], wx2 * wy2, out);
                out = fmaf(r1[x2r], wx1 * wy2, out);
                out = fmaf(r2[x1r], wx2 * wy1, out);
                out = fmaf(r2[x2r], wx1 * wy1, out);
            } else {
                out = out + r1[x1r] * (wx2 * wy2);
                out = out + r1[x2r] * (wx1 * wy2);
                out = out + r2[x1r] * (wx2 * wy1);
                out = out + r2[x2r] * (wx1 * wy1);
            }
            dst[(size_t)y * dw + x] = mul != 1.f ? out * mul : out;
        }
    }
}

/* ---- level image: separable REFLECT101 blur of the full frame (taps g[0..kh]), then the bilinear resize
 * (farneback_gpu_model._sep_filter + resize_linear; k_farn_blur_v4 + k_farn_blur_h_resize).  The blur's tap chain
 * has a run-time length: a plain product first, then one multiply-add per pair. ---- */
int farneback_model_level_image(const float *src, int rows, int cols, const float *g, int kh, int h, int w,
                                float *out) {
    float *V = (float *)malloc(sizeof(float) * (size_t)rows * cols);
    float *B = (float *)malloc(sizeof(float) * (size_t)rows * cols);
    if (!V || !B) {
        free(V);
        free(B);
        return -1;
    }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < rows; ++y) {
        for (int x = 0; x < cols; ++x) {
            float acc = src[(size_t)y * cols + x] * g[0];
            for (int j = 1; j <= kh; ++j)
                acc = mad(src[(size_t)pyr_reflect101(y - j, rows) * cols + x] +
                              src[(size_t)pyr_reflect101(y + j, rows) * cols + x], g[j], acc);
            V[(size_t)y * cols + x] = acc;
        }
    }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < rows; ++y) {
        const float *v = V + (size_t)y * cols;
        for (int x = 0; x < cols; ++x) {
            float acc = v[x] * g[0];
            for (int i = 1; i <= kh; ++i) acc = mad(v[pyr_reflect101(x - i, cols)] + v[pyr_reflect101(x + i, cols)], g[i], acc);
            B[(size_t)y * cols + x] = acc;
        }
    }
    if (!FARN_SKIP_ZERO || (h == rows && w == cols)) {
        resize_linear(B, rows, cols, out, h, w, 1.f);
    } else {
        /* as resize_linear, without the taps whose weight is zero */
        const float ix = (float)(1.0 / ((double)w / cols)), iy = (float)(1.0 / ((double)h / rows));
#pragma omp parallel for schedule(static)
        for (int y = 0; y < h; ++y) {
            const float sy = (float)y * iy;
            const int y1 = (int)floorf(sy), y2 = y1 + 1;
            const int y1r = mini(y1, rows - 1), y2r = mini(y2, rows - 1);
            const float wy2 = (float)y2 - sy, wy1 = sy - (float)y1;
            for (int x = 0; x < w; ++x) {
                const float sx = (float)x * ix;
                const int x1 = (int)floorf(sx), x2 = x1 + 1;
                const int x1r = mini(x1, cols - 1), x2r = mini(x2, cols - 1);
                const float wx2 = (float)x2 - sx, wx1 = sx - (float)x1;
                const float *r1 = B + (size_t)y1r * cols, *r2 = B + (size_t)y2r * cols;
                float o = 0.f;
                if (FARN_FUSED_RESIZE) {
                    o = fmaf(r1[x1r], wx2 * wy2, o);
                    if (wx1 != 0.f) o = fmaf(r1[x2r], wx1 * wy2, o);
                    if (wy1 != 0.f) {
                        o = fmaf(r2[x1r], wx2 * wy1, o);
                        if (wx1 != 0.f) o = fmaf(r2[x2r], wx1 * wy1, o);
                    }
                } else {
                    o = o + r1[x1r] * (wx2 * wy2);
                    if (wx1 != 0.f) o = o + r1[x2r] * (wx1 * wy2);
                    if (wy1 != 0.f) {
                        o = o + r2[x1r] * (wx2 * wy1);
                        if (wx1 != 0.f) o = o + r2[x2r] * (wx1 * wy1);
                    }
                }
                out[(size_t)y * w + x] = o;
            }
        }
    }
    free(V);
    free(B);
    return 0;
}

/* ---- polynomial expansion (farneback_gpu_model.poly_exp; k_farn_polyexp / _fast).  tabs: g[8], xg[8], xxg[8], ig11,
 * ig03, ig33, ig55.  Replicate border.  R: 5 planes of h x w. ---- */
static void poly_exp(const float *src, int h, int w, int n, const float *tabs, float *R) {
    const float *g = tabs, *xg = tabs + 8, *xxg = tabs + 16;
    const float ig11 = tabs[24], ig03 = tabs[25], ig33 = tabs[26], ig55 = tabs[27];
    const size_t np = (size_t)h * w;
    float *V = (float *)malloc(sizeof(float) * 3 * np);
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w; ++x) {
            const float c = src[(size_t)y * w + x];
            float a0 = c * g[0], a1 = 0.f, a2 = 0.f;
            for (int k = 1; k <= n; ++k) {
                const float t0 = src[(size_t)(y - k < 0 ? 0 : y - k) * w + x];
                const float t1 = src[(size_t)mini(y + k, h - 1) * w + x];
                /* the unrolled chain fuses the centre tap into the first pair: fmaf(c, g0, g1 * (t0 + t1)) */
                a0 = (FARN_FMA && k == 1) ? fmaf(c, g[0], g[1] * (t0 + t1)) : mad(g[k], t0 + t1, a0);
                a1 = mad(xg[k], t1 - t0, a1);
                a2 = mad(xxg[k], t0 + t1, a2);
            }
            V[(size_t)y * w + x] = a0;
            V[np + (size_t)y * w + x] = a1;
            V[2 * np + (size_t)y * w + x] = a2;
        }
    }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        const float *r0 = V + (size_t)y * w, *r1 = V + np + (size_t)y * w, *r2 = V + 2 * np + (size_t)y * w;
        for (int x = 0; x < w; ++x) {
            float b1 = g[0] * r0[x], b3 = g[0] * r1[x], b5 = g[0] * r2[x];
            float b2 = 0.f, b4 = 0.f, b6 = 0.f;
            for (int k = 1; k <= n; ++k) {
                const int xa = mini(x + k, w - 1), xb = x - k < 0 ? 0 : x - k;
                const float s0 = r0[xa] + r0[xb], d0 = r0[xa] - r0[xb];
                const float s1 = r1[xa] + r1[xb], d1 = r1[xa] - r1[xb];
                const float s2 = r2[xa] + r2[xb];
                if (FARN_FMA && k == 1) {
                    b1 = fmaf(g[0], r0[x], s0 * g[1]);
                    b3 = fmaf(g[0], r1[x], s1 * g[1]);
                    b5 = fmaf(g[0], r2[x], s2 * g[1]);
                } else {
                    b1 = mad(s0, g[k], b1);
                    b3 = mad(s1, g[k], b3);
                    b5 = mad(s2, g[k], b5);
                }
                b4 = mad(s0, xxg[k], b4);
                b2 = mad(d0, xg[k], b2);
                b6 = mad(d1, xg[k], b6);
            }
            const size_t i = (size_t)y * w + x;
            R[i] = b3 * ig11;
            R[np + i] = b2 * ig11;
            if (FARN_FMA) {
                R[2 * np + i] = fmaf(b1, ig03, b5 * ig33);
                R[3 * np + i] = fmaf(b1, ig03, b4 * ig33);
            } else {
                R[2 * np + i] = b1 * ig03 + b5 * ig33;
                R[3 * np + i] = b1 * ig03 + b4 * ig33;
            }
            R[4 * np + i] = b6 * ig55;
        }
    }
    free(V);
}

static float border_w(int d) { return d <= 1 ? 0.14f : (d < BORDER_SIZE ? 0.4472f : 1.f); }

/* ---- updateMatrices (farneback_gpu_model.update_matrices; farn_update_matrices_px / _quad / _spread) ---- */
static void update_matrices(const float *fxp, const float *fyp, const float *R0, const float *R1, int h, int w,
                            float *M) {
    const size_t np = (size_t)h * w;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w; ++x) {
            const size_t i = (size_t)y * w + x;
            const float dx = fxp[i], dy = fyp[i];
            float fx = (float)x + dx, fy = (float)y + dy;
            long long x1, y1;
            if (FARN_FLOOR_CLAMP) {
                x1 = (int)fminf(fmaxf(floorf(fx), -4.f), (float)w + 4.f);
                y1 = (int)fminf(fmaxf(floorf(fy), -4.f), (float)h + 4.f);
            } else {  /* numpy's float -> int64 conversion: out of range and NaN give INT64_MIN */
                const float a = floorf(fx), b = floorf(fy);
                x1 = (a >= -9.2e18f && a <= 9.2e18f) ? (long long)a : INT64_MIN;
                y1 = (b >= -9.2e18f && b <= 9.2e18f) ? (long long)b : INT64_MIN;
            }
            fx = fx - floorf(fx);
            fy = fy - floorf(fy);
            const int inb = x1 >= 0 && y1 >= 0 && x1 < w - 1 && y1 < h - 1;
            float gth[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
            if (inb) {
                const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy);
                const float a10 = (1.f - fx) * fy, a11 = fx * fy;
                for (int k = 0; k < 5; ++k) {
                    const float *p = R1 + k * np + (size_t)y1 * w + x1;
                    if (FARN_FMA)
                        gth[k] = fmaf(a11, p[w + 1], fmaf(a10, p[w], fmaf(a00, p[0], a01 * p[1])));
                    else
                        gth[k] = a00 * p[0] + a01 * p[1] + a10 * p[w] + a11 * p[w + 1];
                }
            }
            float r2, r3, r4, r5, r6;
            if (inb) {
                r2 = gth[0];
                r3 = gth[1];
                r4 = (R0[2 * np + i] + gth[2]) * 0.5f;
                r5 = (R0[3 * np + i] + gth[3]) * 0.5f;
                r6 = (R0[4 * np + i] + gth[4]) * 0.25f;
            } else {
                r2 = r3 = 0.f;
                r4 = R0[2 * np + i];
                r5 = R0[3 * np + i];
                r6 = R0[4 * np + i] * 0.5f;
            }
            if (FARN_FMA) {  /* r2 = (R0 - r2) * 0.5f; r2 += r4 * dy + r6 * dx; r3 likewise, but nvcc fuses its SECOND
                                product there (r6 * dy rounds, r5 * dx is fused) */
                r2 = fmaf(R0[i] - r2, 0.5f, fmaf(r4, dy, r6 * dx));
                r3 = fmaf(R0[np + i] - r3, 0.5f, fmaf(r5, dx, r6 * dy));
            } else {
                r2 = (R0[i] - r2) * 0.5f;
                r3 = (R0[np + i] - r3) * 0.5f;
                r2 = r2 + r4 * dy + r6 * dx;
                r3 = r3 + r6 * dy + r5 * dx;
            }
            const float scale = border_w(mini(x, BORDER_SIZE)) * border_w(mini(y, BORDER_SIZE)) *
                                border_w(mini(w - x - 1, BORDER_SIZE)) * border_w(mini(h - y - 1, BORDER_SIZE));
            r2 *= scale;
            r3 *= scale;
            r4 *= scale;
            r5 *= scale;
            r6 *= scale;
            if (FARN_FMA) {
                M[i] = fmaf(r4, r4, r6 * r6);
                M[2 * np + i] = fmaf(r5, r5, r6 * r6);
                M[3 * np + i] = fmaf(r4, r2, r6 * r3);
                M[4 * np + i] = fmaf(r6, r2, r5 * r3);
            } else {
                M[i] = r4 * r4 + r6 * r6;
                M[2 * np + i] = r5 * r5 + r6 * r6;
                M[3 * np + i] = r4 * r2 + r6 * r3;
                M[4 * np + i] = r6 * r2 + r5 * r3;
            }
            M[np + i] = (r4 + r5) * r6;
        }
    }
}

/* balanced tree over 13 values (farneback.cu box_first) */
static inline float box_first13(const float *v) {
    const float a = (v[0] + v[1]) + (v[2] + v[3]), b = (v[4] + v[5]) + (v[6] + v[7]);
    const float c = (v[8] + v[9]) + (v[10] + v[11]);
    return ((a + b) + c) + v[12];
}

/* ---- the window blur of one plane, replicate border (farneback_gpu_model.box_filter5 / _sep_filter; the vertical and
 * horizontal passes of k_farn_iter, k_farn_iter_fast, k_farn_iter_tma).  taps == NULL: box; box_inv scales the box
 * sum.  V: h x w scratch. ---- */
static void window_blur(const float *P, int h, int w, int k, const float *taps, float box_inv, int order, float *V,
                        float *out) {
    const int running = FARN_RUNNING_BOX && !taps && order == ORDER_FAST && k == 6;
    const int fused_first = FARN_FMA && taps && order == ORDER_FAST && k == 6;
    if (running) {
        const int strips = (h + 15) / 16;
#pragma omp parallel for schedule(static)
        for (int s = 0; s < strips; ++s) {
            const int y0 = 16 * s;
            for (int x = 0; x < w; ++x) {
                float v[28];
                for (int q = 0; q < 28; ++q) v[q] = P[(size_t)clampi(y0 - 6 + q, 0, h - 1) * w + x];
                float acc = box_first13(v);
                for (int o = 0; o < 16 && y0 + o < h; ++o) {
                    if (o) acc = acc + (v[o + 12] - v[o - 1]);
                    V[(size_t)(y0 + o) * w + x] = acc;
                }
            }
        }
#pragma omp parallel for schedule(static)
        for (int y = 0; y < h; ++y) {
            const float *r = V + (size_t)y * w;
            for (int x0 = 0; x0 < w; x0 += 4) {
                float c[16];
                for (int q = 0; q < 16; ++q) c[q] = r[clampi(x0 - 6 + q, 0, w - 1)];
                float acc = box_first13(c);
                for (int e = 0; e < 4 && x0 + e < w; ++e) {
                    if (e) acc = acc + (c[e + 12] - c[e - 1]);
                    out[(size_t)y * w + x0 + e] = acc * box_inv;
                }
            }
        }
        return;
    }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w; ++x) {
            const float c = P[(size_t)y * w + x];
            float acc = taps ? c * taps[0] : c;
            for (int j = 1; j <= k; ++j) {
                const float s = P[(size_t)(y - j < 0 ? 0 : y - j) * w + x] + P[(size_t)mini(y + j, h - 1) * w + x];
                if (!taps) acc = acc + s;
                else if (fused_first && j == 1) acc = fmaf(c, taps[0], s * taps[1]);
                else acc = mad(s, taps[j], acc);
            }
            V[(size_t)y * w + x] = acc;
        }
    }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        const float *r = V + (size_t)y * w;
        for (int x = 0; x < w; ++x) {
            float acc = taps ? r[x] * taps[0] : r[x];
            for (int i = 1; i <= k; ++i) {
                const float s = r[x - i < 0 ? 0 : x - i] + r[mini(x + i, w - 1)];
                if (!taps) acc = acc + s;
                else if (fused_first && i == 1) acc = fmaf(r[x], taps[0], s * taps[1]);
                else acc = mad(s, taps[i], acc);
            }
            out[(size_t)y * w + x] = taps ? acc : acc * box_inv;
        }
    }
}

/* the box filter alone (5 planes), for tests of the summation order */
void farneback_model_box(const float *M, int h, int w, int win_size, int order, float *out) {
    const int k = win_size / 2;
    float *V = (float *)malloc(sizeof(float) * (size_t)h * w);
    const float box_inv = 1.f / (float)((1 + 2 * k) * (1 + 2 * k));
    for (int p = 0; p < 5; ++p)
        window_blur(M + (size_t)p * h * w, h, w, k, NULL, box_inv, order, V, out + (size_t)p * h * w);
    free(V);
}

/* ---- updateFlow (farneback_gpu_model.update_flow; the 2x2 solve of every iteration kernel) ---- */
static void update_flow(const float *B, int h, int w, float *fx, float *fy) {
    const size_t np = (size_t)h * w;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w; ++x) {
            const size_t i = (size_t)y * w + x;
            const float g11 = B[i], g12 = B[np + i], g22 = B[2 * np + i], h1 = B[3 * np + i], h2 = B[4 * np + i];
            if (FARN_FMA) {
                const float det_inv = 1.f / (fmaf(g11, g22, -(g12 * g12)) + 1e-3f);
                fx[i] = fmaf(g11, h2, -(g12 * h1)) * det_inv;
                fy[i] = fmaf(g22, h1, -(g12 * h2)) * det_inv;
            } else {
                const float det_inv = 1.f / (g11 * g22 - g12 * g12 + 1e-3f);
                fx[i] = (g11 * h2 - g12 * h1) * det_inv;
                fy[i] = (g22 * h1 - g12 * h2) * det_inv;
            }
        }
    }
}

static int cv_round(double v) { return (int)nearbyint(v); }

/* farneback_gpu_model.calc.  I0, I1: rows x cols float frames (u8 converted without scaling).  poly_tabs: 28 floats
 * (see poly_exp).  img_taps + img_taps_off[k] .. img_taps_off[k + 1]: the half level-image kernel of level k (unused with
 * fast_pyramids).  win_taps: the half window kernel (GAUSSIAN flag).  pyr_in: with fast_pyramids and without
 * FARN_PYR_TAP5, levels 1.. of frame 0 then of frame 1, concatenated.  init_flow: interleaved rows x cols x 2 (flag
 * USE_INITIAL_FLOW).  order: ORDER_FAST / ORDER_GENERIC.  flow: interleaved rows x cols x 2.
 * Returns 0, -1 when out of memory, -2 on a bad argument. */
int farneback_model_calc(const float *I0, const float *I1, int rows, int cols, int num_levels, double pyr_scale,
                         int fast_pyramids, int win_size, int num_iters, int poly_n, int flags, const float *poly_tabs,
                         const float *img_taps, const int *img_taps_off, const float *win_taps, const float *pyr_in,
                         const float *init_flow, int order, float *flow) {
    if (rows < 1 || cols < 1 || !(poly_n == 5 || poly_n == 7) || win_size < 1 || !(win_size & 1) || num_iters < 0)
        return -2;
    int cropped = 0;
    double scale = 1;
    for (; cropped < num_levels; ++cropped) {
        scale *= pyr_scale;
        if (cols * scale < MIN_SIZE || rows * scale < MIN_SIZE) break;
    }
    if (cropped >= MAX_LEVELS) return -2;
    int lh[MAX_LEVELS], lw[MAX_LEVELS];
    double lscale[MAX_LEVELS];
    for (int k = 0; k <= cropped; ++k) {
        double s = 1;
        for (int i = 0; i < k; ++i) s *= pyr_scale;
        lscale[k] = s;
        if (fast_pyramids) {
            lh[k] = k ? (lh[k - 1] + 1) / 2 : rows;
            lw[k] = k ? (lw[k - 1] + 1) / 2 : cols;
        } else {
            lh[k] = cv_round(rows * s);
            lw[k] = cv_round(cols * s);
        }
    }
    const size_t N = (size_t)rows * cols;
    float *pyr[2][MAX_LEVELS] = {{0}};
    float *img[2] = {0}, *R[2] = {0}, *M = 0, *B = 0, *V = 0, *fx = 0, *fy = 0, *pfx = 0, *pfy = 0;
    int rc = 0;
    img[0] = malloc(sizeof(float) * N);
    img[1] = malloc(sizeof(float) * N);
    R[0] = malloc(sizeof(float) * 5 * N);
    R[1] = malloc(sizeof(float) * 5 * N);
    M = malloc(sizeof(float) * 5 * N);
    B = malloc(sizeof(float) * 5 * N);
    V = malloc(sizeof(float) * N);
    fx = malloc(sizeof(float) * N);
    fy = malloc(sizeof(float) * N);
    pfx = malloc(sizeof(float) * N);
    pfy = malloc(sizeof(float) * N);
    if (!img[0] || !img[1] || !R[0] || !R[1] || !M || !B || !V || !fx || !fy || !pfx || !pfy) {
        rc = -1;
        goto done;
    }
    if (fast_pyramids) {
        const float *src = pyr_in;
        for (int i = 0; i < 2; ++i) {
            pyr[i][0] = (float *)(i ? I1 : I0);
            for (int k = 1; k <= cropped; ++k) {
                pyr[i][k] = malloc(sizeof(float) * (size_t)lh[k] * lw[k]);
                if (!pyr[i][k]) {
                    rc = -1;
                    goto done;
                }
                if (FARN_PYR_TAP5) {
                    if (pyr_tap5_down(pyr[i][k - 1], lh[k - 1], lw[k - 1], pyr[i][k])) {
                        rc = -1;
                        goto done;
                    }
                } else {
                    if (!src) {
                        rc = -2;
                        goto done;
                    }
                    memcpy(pyr[i][k], src, sizeof(float) * (size_t)lh[k] * lw[k]);
                    src += (size_t)lh[k] * lw[k];
                }
            }
        }
    }
    const int k_win = win_size / 2;
    /* the engine's float reciprocal; it equals the numpy model's float(1 / area) for every window */
    const float box_inv = 1.f / (float)((1 + 2 * k_win) * (1 + 2 * k_win));
    for (int k = cropped; k >= 0; --k) {
        const int h = lh[k], w = lw[k];
        const size_t np = (size_t)h * w;
        if (k == cropped) {
            if (flags & USE_INITIAL_FLOW) {
                for (size_t i = 0; i < N; ++i) {
                    pfx[i] = init_flow[2 * i];
                    pfy[i] = init_flow[2 * i + 1];
                }
                resize_linear(pfx, rows, cols, fx, h, w, (float)lscale[k]);
                resize_linear(pfy, rows, cols, fy, h, w, (float)lscale[k]);
            } else {
                memset(fx, 0, sizeof(float) * np);
                memset(fy, 0, sizeof(float) * np);
            }
        } else {
            memcpy(pfx, fx, sizeof(float) * (size_t)lh[k + 1] * lw[k + 1]);
            memcpy(pfy, fy, sizeof(float) * (size_t)lh[k + 1] * lw[k + 1]);
            resize_linear(pfx, lh[k + 1], lw[k + 1], fx, h, w, (float)(1. / pyr_scale));
            resize_linear(pfy, lh[k + 1], lw[k + 1], fy, h, w, (float)(1. / pyr_scale));
        }
        for (int i = 0; i < 2; ++i) {
            const float *lvl;
            if (fast_pyramids) {
                lvl = pyr[i][k];
            } else {
                const int kh = img_taps_off[k + 1] - img_taps_off[k] - 1;
                if (farneback_model_level_image(i ? I1 : I0, rows, cols, img_taps + img_taps_off[k], kh, h, w, img[i])) {
                    rc = -1;
                    goto done;
                }
                lvl = img[i];
            }
            poly_exp(lvl, h, w, poly_n, poly_tabs, R[i]);
        }
        update_matrices(fx, fy, R[0], R[1], h, w, M);
        for (int it = 0; it < num_iters; ++it) {
            for (int p = 0; p < 5; ++p)
                window_blur(M + p * np, h, w, k_win, (flags & GAUSSIAN) ? win_taps : NULL, box_inv, order, V, B + p * np);
            update_flow(B, h, w, fx, fy);
            if (it < num_iters - 1) update_matrices(fx, fy, R[0], R[1], h, w, M);
        }
    }
    for (size_t i = 0; i < N; ++i) {
        flow[2 * i] = fx[i];
        flow[2 * i + 1] = fy[i];
    }
done:
    for (int i = 0; i < 2; ++i)
        for (int k = 1; k <= cropped; ++k) free(pyr[i][k]);
    free(img[0]);
    free(img[1]);
    free(R[0]);
    free(R[1]);
    free(M);
    free(B);
    free(V);
    free(fx);
    free(fy);
    free(pfx);
    free(pfy);
    return rc;
}
