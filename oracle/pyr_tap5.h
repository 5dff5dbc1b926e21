/* pyr_tap5.h -- the engine's pyrDown (opencv_contrib_b200/csrc/pyramid.cu k_pyr_down<false>, pyr_tap5) restated in C,
 * shared by the C models that build fastPyramids / DensePyrLK pyramids.  TEST INFRASTRUCTURE; compile with
 * -ffp-contract=off so that fmaf() stands exactly where pyr_tap5 fuses and every other operation rounds on its own. */
#ifndef ORACLE_PYR_TAP5_H
#define ORACLE_PYR_TAP5_H

#include <math.h>
#include <stdlib.h>

/* BORDER_REFLECT101 index: -1 -> 1, n -> n-2 */
static inline int pyr_reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        if (i >= n) i = 2 * n - 2 - i;
    }
    return i;
}

/* pyramid.cu pyr_tap5: the first two products summed with one rounding, then one fused multiply-add per tap */
static inline float pyr_tap5(float a, float b, float c, float d, float e) {
    float s = fmaf(a, 0.0625f, b * 0.25f);
    s = fmaf(c, 0.375f, s);
    s = fmaf(d, 0.25f, s);
    return fmaf(e, 0.0625f, s);
}

/* k_pyr_down<false>: vertical 5-tap per source column, then horizontal, REFLECT101; dst is ((h+1)/2, (w+1)/2).
 * Returns 0, or -1 when out of memory. */
static inline int pyr_tap5_down(const float *src, int h, int w, float *dst) {
    const int dh = (h + 1) / 2, dw = (w + 1) / 2;
    float *V = (float *)malloc(sizeof(float) * (size_t)dh * w);
    if (!V) return -1;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < dh; ++y) {
        const float *r[5];
        for (int k = 0; k < 5; ++k) r[k] = src + (size_t)pyr_reflect101(2 * y - 2 + k, h) * w;
        for (int x = 0; x < w; ++x) V[(size_t)y * w + x] = pyr_tap5(r[0][x], r[1][x], r[2][x], r[3][x], r[4][x]);
    }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < dh; ++y) {
        const float *v = V + (size_t)y * w;
        for (int x = 0; x < dw; ++x) {
            int rx[5];
            for (int k = 0; k < 5; ++k) rx[k] = pyr_reflect101(2 * x - 2 + k, w);
            dst[(size_t)y * dw + x] = pyr_tap5(v[rx[0]], v[rx[1]], v[rx[2]], v[rx[3]], v[rx[4]]);
        }
    }
    free(V);
    return 0;
}

#endif
