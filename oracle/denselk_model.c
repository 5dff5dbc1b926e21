/* denselk_model.c -- C/OpenMP restatement of oracle/denselk_model.py, operation for operation, so that the
 * DensePyrLK engine (opencv_contrib_b200/csrc/denselk.cu, pyramid.cu) can be compared with it bit for bit at full
 * frame size.  TEST INFRASTRUCTURE (see oracle/__init__.py); never linked into libb200flow.so.
 *
 * Built with -ffp-contract=off: every float operation rounds on its own, and fmaf() stands exactly where the
 * kernels fuse (pyr_tap5, lk_scharr3, D, dx, dy, the initial track).  int32 accumulators wrap around through
 * unsigned arithmetic, as in the kernels.  Rows are independent within a level: OpenMP over rows. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "pyr_tap5.h"

enum { MAX_WIN = 256 }; /* the engine's 200 KB patch limit allows windows up to 115 */
enum { C_WRAPPED, C_SINGULAR, C_LEFT, C_CAPPED, C_CHAIN, N_COUNTERS };

int denselk_model_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
#else
    (void)n;
    return 1;
#endif
}

int denselk_model_n_counters(void) { return N_COUNTERS; }

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* k_pyr_down<false> (pyr_tap5.h, shared with farneback_model.c) */
void denselk_model_pyr_down(const float *src, int h, int w, float *dst) { (void)pyr_tap5_down(src, h, w, dst); }

/* denselk.cu lk_scharr3 */
static float scharr3(float a, float b, float c) { return fmaf(c, 3.f, fmaf(a, 3.f, 10.f * b)); }

/* denselk.cu lk_axis */
static void lk_axis(float coord, int n, int *ia, int *ic, float *a) {
    const float b = coord - 0.5f;
    const float f = floorf(b);
    *a = floorf((b - f) * 256.f + 0.5f) * (1.f / 256.f);
    const int i0 = (int)fminf(fmaxf(f, -2.f), (float)n + 1.f);
    *ia = clampi(i0, 0, n - 1);
    *ic = clampi(i0 + 1, 0, n - 1);
}

static float lk_blend(float ax, float ay, float t00, float t01, float t10, float t11) {
    const float bx = 1.f - ax, by = 1.f - ay;
    float r = (bx * by) * t00;
    r = r + (ax * by) * t01;
    r = r + (bx * ay) * t10;
    r = r + (ax * ay) * t11;
    return r;
}

static int outside32(int64_t v) { return v < INT32_MIN || v > INT32_MAX; }

/* k_lk_dense for one level.  u, v, prevU, prevV: full-resolution planes with row stride `stride`. */
static void level(const float *I, const float *J, int h, int w, float *u, float *v, const float *prevU, const float *prevV,
                  int stride, int wx, int wy, int iters, long long *cnt) {
    const int hx = (wx - 1) / 2, hy = (wy - 1) / 2;
    const int EW = w + wx - 1, EH = h + wy - 1;
    /* patch cell (i, j) of pixel (y, x) holds the values at texel (y - hy + i, x - hx + j) */
    int *Ip = (int *)malloc(sizeof(int) * (size_t)EH * EW);
    int *gx = (int *)malloc(sizeof(int) * (size_t)EH * EW);
    int *gy = (int *)malloc(sizeof(int) * (size_t)EH * EW);
#pragma omp parallel for schedule(static)
    for (int ey = 0; ey < EH; ++ey) {
        for (int ex = 0; ex < EW; ++ex) {
            const int py = ey - hy, px = ex - hx;
#define T(dy, dx) I[(size_t)clampi(py + (dy), 0, h - 1) * w + clampi(px + (dx), 0, w - 1)]
            const size_t e = (size_t)ey * EW + ex;
            Ip[e] = (int)T(0, 0);
            gx[e] = (int)(scharr3(T(-1, 1), T(0, 1), T(1, 1)) - scharr3(T(-1, -1), T(0, -1), T(1, -1)));
            gy[e] = (int)(scharr3(T(1, -1), T(1, 0), T(1, 1)) - scharr3(T(-1, -1), T(-1, 0), T(-1, 1)));
#undef T
        }
    }
    long long c_wrapped = 0, c_singular = 0, c_left = 0, c_capped = 0, c_chain = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : c_wrapped, c_singular, c_left, c_capped, c_chain)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w; ++x) {
            int64_t s11 = 0, s12 = 0, s22 = 0;
            for (int i = 0; i < wy; ++i) {
                const size_t e = (size_t)(y + i) * EW + x;
                for (int j = 0; j < wx; ++j) {
                    const int64_t dx = gx[e + j], dy = gy[e + j];
                    s11 += dx * dx;
                    s12 += dx * dy;
                    s22 += dy * dy;
                }
            }
            c_wrapped += outside32(s11) + outside32(s12) + outside32(s22);
            float A11 = (float)(int32_t)(uint32_t)s11, A12 = (float)(int32_t)(uint32_t)s12;
            float A22 = (float)(int32_t)(uint32_t)s22;
            float D = fmaf(A11, A22, -(A12 * A12));
            if (D < FLT_EPSILON) {
                ++c_singular;
                continue;
            }
            D = 1.f / D;
            A11 = A11 * D;
            A12 = A12 * D;
            A22 = A22 * D;
            float nx = fmaf(prevU[(size_t)(y / 2) * stride + x / 2], 2.0f, (float)x);
            float ny = fmaf(prevV[(size_t)(y / 2) * stride + x / 2], 2.0f, (float)y);
            int left = 0, converged = 0;
            for (int k = 0; k < iters; ++k) {
                if (nx < 0 || nx >= w || ny < 0 || ny >= h) {
                    left = 1;
                    break;
                }
                int xap[MAX_WIN], xcp[MAX_WIN];
                float axp[MAX_WIN];
                int chained = 1;
                for (int j = 0; j < wx; ++j) {
                    lk_axis(((nx - (float)hx) + (float)j) + 0.5f, w, &xap[j], &xcp[j], &axp[j]);
                    if (j > 0 && xap[j] != xcp[j - 1]) chained = 0;
                }
                if (wx == 13 && !chained) ++c_chain;
                int64_t b1 = 0, b2 = 0;
                for (int i = 0; i < wy; ++i) {
                    int ya, yc;
                    float ay;
                    lk_axis(((ny - (float)hy) + (float)i) + 0.5f, h, &ya, &yc, &ay);
                    const float *ra = J + (size_t)ya * w, *rc = J + (size_t)yc * w;
                    const size_t e = (size_t)(y + i) * EW + x;
                    for (int j = 0; j < wx; ++j) {
                        const int Jv = (int)lk_blend(axp[j], ay, ra[xap[j]], ra[xcp[j]], rc[xap[j]], rc[xcp[j]]);
                        const int64_t diff = (int64_t)(Jv - Ip[e + j]) * 32;
                        b1 += diff * gx[e + j];
                        b2 += diff * gy[e + j];
                    }
                }
                c_wrapped += outside32(b1) + outside32(b2);
                const float fb1 = (float)(int32_t)(uint32_t)b1, fb2 = (float)(int32_t)(uint32_t)b2;
                const float dx = fmaf(A12, fb2, -(A22 * fb1));
                const float dy = fmaf(A12, fb1, -(A11 * fb2));
                nx = nx + dx;
                ny = ny + dy;
                if (fabsf(dx) < 0.01f && fabsf(dy) < 0.01f) {
                    converged = 1;
                    break;
                }
            }
            if (left) {
                ++c_left;
                continue;
            }
            if (!converged) ++c_capped;
            u[(size_t)y * stride + x] = nx - (float)x;
            v[(size_t)y * stride + x] = ny - (float)y;
        }
    }
    cnt[C_WRAPPED] += c_wrapped;
    cnt[C_SINGULAR] += c_singular;
    cnt[C_LEFT] += c_left;
    cnt[C_CAPPED] += c_capped;
    cnt[C_CHAIN] += c_chain;
    free(Ip);
    free(gx);
    free(gy);
}

/* denselk_model.calc: uint8 frames in, interleaved (rows, cols, 2) float flow out.  counters: (max_level + 1) *
 * N_COUNTERS entries, coarsest level first.  Returns 0, -1 when out of memory, -2 on a bad argument. */
int denselk_model_calc(const unsigned char *I0, const unsigned char *I1, int rows, int cols, int win_x, int win_y,
                       int max_level, int iters, float *flow, long long *counters) {
    if (rows < 1 || cols < 1 || win_x < 1 || win_x > MAX_WIN || win_y < 1 || max_level < 0 || iters < 0) return -2;
    float **pI = (float **)calloc(max_level + 1, sizeof(float *)), **pJ = (float **)calloc(max_level + 1, sizeof(float *));
    int *lh = (int *)malloc(sizeof(int) * (max_level + 1)), *lw = (int *)malloc(sizeof(int) * (max_level + 1));
    const size_t n = (size_t)rows * cols;
    float *uP[2], *vP[2];
    for (int i = 0; i < 2; ++i) {
        uP[i] = (float *)calloc(n, sizeof(float));
        vP[i] = (float *)calloc(n, sizeof(float));
    }
    int rc = 0;
    if (!pI || !pJ || !lh || !lw || !uP[0] || !uP[1] || !vP[0] || !vP[1]) {
        rc = -1;
        goto done;
    }
    lh[0] = rows;
    lw[0] = cols;
    pI[0] = (float *)malloc(sizeof(float) * n);
    pJ[0] = (float *)malloc(sizeof(float) * n);
    if (!pI[0] || !pJ[0]) {
        rc = -1;
        goto done;
    }
    for (size_t i = 0; i < n; ++i) {
        pI[0][i] = (float)I0[i];
        pJ[0][i] = (float)I1[i];
    }
    for (int l = 1; l <= max_level; ++l) {
        lh[l] = (lh[l - 1] + 1) / 2;
        lw[l] = (lw[l - 1] + 1) / 2;
        pI[l] = (float *)malloc(sizeof(float) * (size_t)lh[l] * lw[l]);
        pJ[l] = (float *)malloc(sizeof(float) * (size_t)lh[l] * lw[l]);
        if (!pI[l] || !pJ[l]) {
            rc = -1;
            goto done;
        }
        denselk_model_pyr_down(pI[l - 1], lh[l - 1], lw[l - 1], pI[l]);
        denselk_model_pyr_down(pJ[l - 1], lh[l - 1], lw[l - 1], pJ[l]);
    }
    memset(counters, 0, sizeof(long long) * N_COUNTERS * (max_level + 1));
    int idx = 0;
    for (int l = max_level; l >= 0; --l) {
        const int idx2 = (idx + 1) & 1;
        level(pI[l], pJ[l], lh[l], lw[l], uP[idx], vP[idx], uP[idx2], vP[idx2], cols, win_x, win_y, iters,
              counters + (size_t)(max_level - l) * N_COUNTERS);
        if (l > 0) idx = idx2;
    }
    for (size_t i = 0; i < n; ++i) {
        flow[2 * i] = uP[idx][i];
        flow[2 * i + 1] = vP[idx][i];
    }
done:
    for (int l = 0; l <= max_level && pI && pJ; ++l) {
        free(pI[l]);
        free(pJ[l]);
    }
    free(pI);
    free(pJ);
    free(lh);
    free(lw);
    for (int i = 0; i < 2; ++i) {
        free(uP[i]);
        free(vP[i]);
    }
    return rc;
}
