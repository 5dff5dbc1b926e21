/* superres_model.c -- the BTV-L1 super-resolution step of cv::superres::createSuperResolution_BTVL1_CUDA
 * (modules/superres/src/btv_l1_cuda.cpp:306-400, src/cuda/btv_l1_gpu.cu), restated operation by operation and unfused:
 * every full-resolution intermediate the reference allocates is computed whole, in the reference's order.
 * TEST INFRASTRUCTURE (see oracle/__init__.py); never linked into libb200flow.so.
 *
 * Float only, built with -ffp-contract=off: every operator rounds once (the engine is built with -fmad=false).  The
 * reference's own contraction of its cubic, filter and addWeighted sums depends on its build; this model picks one
 * rounding per operator.  Formulas of core's headers, which are not in the reference tree:
 *   CubicFilter     taps ceil(c - 2) .. floor(c + 2), Keys a = -0.5, sum w v / sum w, replicated border
 *   PointFilter     src(clamp(trunc(y)), clamp(trunc(x)))
 *   convertTo(8U)   round half to even, saturate
 * Layouts: images H x W x C interleaved, flow planes H x W, all contiguous. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* cudafilters' reflect-101 (BrdRowReflect101::idx_col_low below the image, idx_col_high above it) */
static int reflect101(int x, int n) {
    const int last = n - 1;
    if (x < 0) return abs(x) % n;
    if (x > last) return abs(last - abs(last - x)) % n;
    return x;
}

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* __float2int_rz: truncation, NaN -> 0, saturating */
static int f2i_rz(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return 2147483647;
    if (v <= -2147483648.0f) return (int)-2147483647 - 1;
    return (int)v;
}

static float cubic_coeff(float x_) {
    const float x = fabsf(x_);
    if (x <= 1.0f) return x * x * (1.5f * x - 2.5f) + 1.0f;
    if (x < 2.0f) return x * (x * (-0.5f * x + 2.5f) - 4.0f) + 2.0f;
    return 0.0f;
}

static float diff_sign(float a, float b) { return a > b ? 1.0f : a < b ? -1.0f : 0.0f; }

/* cvtColor(BGR2GRAY / BGRA2GRAY) with cudev's 15-bit rule, then convertTo(CV_32F, 1/255) when to_f32 */
void sr_model_gray(const uint8_t *src, int rows, int cols, int cn, int to_f32, void *dst) {
    for (long i = 0; i < (long)rows * cols; ++i) {
        const uint8_t *p = src + i * cn;
        const int g = cn == 1 ? p[0] : (p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + (1 << 14)) >> 15;
        if (to_f32)
            ((float *)dst)[i] = (float)(1.0 / 255.0) * (float)g;
        else
            ((uint8_t *)dst)[i] = (uint8_t)g;
    }
}

/* getGaussianKernel(n, sigma, CV_32F) */
void sr_model_gaussian_kernel(int n, double sigma, float *out) {
    static const double t1[] = {1.0}, t3[] = {0.25, 0.5, 0.25}, t5[] = {0.0625, 0.25, 0.375, 0.25, 0.0625},
                        t7[] = {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125},
                        t9[] = {4 / 256.0, 13 / 256.0, 30 / 256.0, 51 / 256.0, 60 / 256.0, 51 / 256.0, 30 / 256.0, 13 / 256.0,
                                4 / 256.0};
    const double *tab = n == 1 ? t1 : n == 3 ? t3 : n == 5 ? t5 : n == 7 ? t7 : n == 9 ? t9 : NULL;
    if (tab && sigma <= 0) {
        for (int i = 0; i < n; ++i) out[i] = (float)tab[i];
        return;
    }
    const double sx = sigma > 0 ? sigma : fma((double)n, 0.15, 0.35);
    const double scale2 = -0.125 / (sx * sx);
    const int h = (n - 1) / 2;
    double v[64], sum = 0;
    for (int i = 0, x = 1 - n; i < h; ++i, x += 2) {
        v[i] = exp((double)(x * x) * scale2);
        sum += v[i];
    }
    sum *= 2;
    sum += 1;
    if ((n & 1) == 0) sum += 1;
    const double mul = 1.0 / sum;
    for (int i = 0; i < h; ++i) out[i] = out[n - 1 - i] = (float)(v[i] * mul);
    out[h] = (float)(1.0 * mul);
    if ((n & 1) == 0) out[h + 1] = out[h];
}

/* cuda::createGaussianFilter(...)->apply: the row filter into a float buffer, then the column filter; each tap
 * sum = sum + src * kernel[k], k ascending, anchor n / 2, reflect-101 */
void sr_model_sep_filter(const float *src, int H, int W, int C, const float *k, int n, float *dst) {
    float *buf = malloc(sizeof(float) * (size_t)H * W * C);
    const int an = n / 2;
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
            for (int c = 0; c < C; ++c) {
                float sum = 0.0f;
                for (int i = 0; i < n; ++i) sum = sum + src[((size_t)y * W + reflect101(x - an + i, W)) * C + c] * k[i];
                buf[((size_t)y * W + x) * C + c] = sum;
            }
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
            for (int c = 0; c < C; ++c) {
                float sum = 0.0f;
                for (int j = 0; j < n; ++j) sum = sum + buf[((size_t)reflect101(y - an + j, H) * W + x) * C + c] * k[j];
                dst[((size_t)y * W + x) * C + c] = sum;
            }
    free(buf);
}

/* cuda::resize(src, dst, (W s, H s), INTER_CUBIC): kernel scale float(1 / s), samples at p * fx, top-left aligned */
static void resize_cubic(const float *src, int H, int W, int C, int s, float *dst) {
    const float inv = (float)(1.0 / s);
    const int HH = H * s, WW = W * s;
    for (int y = 0; y < HH; ++y)
        for (int x = 0; x < WW; ++x) {
            const float xc = (float)x * inv, yc = (float)y * inv;
            const float xmin = ceilf(xc - 2.0f), xmax = floorf(xc + 2.0f), ymin = ceilf(yc - 2.0f), ymax = floorf(yc + 2.0f);
            float sum[4] = {0, 0, 0, 0}, wsum = 0.0f;
            for (float cy = ymin; cy <= ymax; cy += 1.0f)
                for (float cx = xmin; cx <= xmax; cx += 1.0f) {
                    const float w = cubic_coeff(xc - cx) * cubic_coeff(yc - cy);
                    const float *p = src + ((size_t)clampi((int)floorf(cy), 0, H - 1) * W + clampi((int)floorf(cx), 0, W - 1)) * C;
                    for (int c = 0; c < C; ++c) sum[c] = sum[c] + w * p[c];
                    wsum += w;
                }
            for (int c = 0; c < C; ++c) dst[((size_t)y * WW + x) * C + c] = wsum == 0.0f ? 0.0f : sum[c] / wsum;
        }
}

/* cuda::remap(src, dst, mapx, mapy, INTER_NEAREST, BORDER_REPLICATE) */
static void remap_nearest(const float *src, int H, int W, int C, const float *mx, const float *my, float *dst) {
    for (size_t i = 0; i < (size_t)H * W; ++i) {
        const int yy = clampi(f2i_rz(my[i]), 0, H - 1), xx = clampi(f2i_rz(mx[i]), 0, W - 1);
        for (int c = 0; c < C; ++c) dst[i * C + c] = src[((size_t)yy * W + xx) * C + c];
    }
}

/* process(src, dst, forwardMotions, backwardMotions, baseIdx) before the crop.
 *   src   K x H x W x C float frames of the window
 *   fwd   K x 2 x H x W: fwd[k] = flow frame k -> k + 1 (k < K - 1)
 *   bwd   K x 2 x H x W: bwd[k] = flow frame k -> k - 1 (k > 0)
 *   hr    out: (H s) x (W s) x C */
int sr_model_process(const float *src, const float *fwd, const float *bwd, int K, int base, int H, int W, int C, int s,
                     int iterations, double tau, double lambda, double alpha, int btv_kernel_size, int blur_kernel_size,
                     double blur_sigma, float *hr) {
    const size_t lp = (size_t)H * W, HH = (size_t)H * s, WW = (size_t)W * s, hp = HH * WW;
    float *relF = calloc(2 * lp * K, sizeof(float)), *relB = calloc(2 * lp * K, sizeof(float));
    float *fmap = malloc(sizeof(float) * 2 * hp * K), *bmap = malloc(sizeof(float) * 2 * hp * K);
    float *up = malloc(sizeof(float) * hp), *a = malloc(sizeof(float) * hp * C), *b = malloc(sizeof(float) * hp * C);
    float *c = malloc(sizeof(float) * lp * C), *diff = malloc(sizeof(float) * hp * C * K), *reg = malloc(sizeof(float) * hp * C);
    float kern[32], w[96];
    if (!relF || !relB || !fmap || !bmap || !up || !a || !b || !c || !diff || !reg) return -1;

    /* 1. calcRelativeMotions (btv_l1_cuda.cpp:80-115): cuda::add outward from baseIdx */
    for (int i = base - 1; i >= 0; --i)
        for (int comp = 0; comp < 2; ++comp)
            for (size_t p = 0; p < lp; ++p) {
                relF[(2 * i + comp) * lp + p] = relF[(2 * (i + 1) + comp) * lp + p] + fwd[(2 * i + comp) * lp + p];
                relB[(2 * i + comp) * lp + p] = relB[(2 * (i + 1) + comp) * lp + p] + bwd[(2 * (i + 1) + comp) * lp + p];
            }
    for (int i = base + 1; i < K; ++i)
        for (int comp = 0; comp < 2; ++comp)
            for (size_t p = 0; p < lp; ++p) {
                relF[(2 * i + comp) * lp + p] = relF[(2 * (i - 1) + comp) * lp + p] + bwd[(2 * i + comp) * lp + p];
                relB[(2 * i + comp) * lp + p] = relB[(2 * (i - 1) + comp) * lp + p] + fwd[(2 * (i - 1) + comp) * lp + p];
            }
    /* 2. upscaleMotions: resize INTER_CUBIC, then multiply(scale); 3. buildMotionMaps: forwardMap = p + backwardMotion,
     *    backwardMap = p + forwardMotion */
    for (int k = 0; k < K; ++k)
        for (int comp = 0; comp < 2; ++comp) {
            resize_cubic(relF + (2 * k + comp) * lp, H, W, 1, s, up);
            for (size_t i = 0; i < hp; ++i) up[i] = up[i] * (float)s;
            for (size_t i = 0; i < hp; ++i)
                bmap[(2 * k + comp) * hp + i] = (float)(comp == 0 ? (int)(i % WW) : (int)(i / WW)) + up[i];
            resize_cubic(relB + (2 * k + comp) * lp, H, W, 1, s, up);
            for (size_t i = 0; i < hp; ++i) up[i] = up[i] * (float)s;
            for (size_t i = 0; i < hp; ++i)
                fmap[(2 * k + comp) * hp + i] = (float)(comp == 0 ? (int)(i % WW) : (int)(i / WW)) + up[i];
        }
    /* 4. initial estimate */
    resize_cubic(src + (size_t)base * lp * C, H, W, C, s, hr);

    sr_model_gaussian_kernel(blur_kernel_size, blur_sigma, kern);
    const int ks = (btv_kernel_size - 1) / 2;
    {
        const float af = (float)alpha;
        for (int m = 0, ind = 0; m <= ks; ++m)
            for (int l = ks; l + m >= 0; --l, ++ind) w[ind] = (float)pow((double)af, (double)(abs(m) + abs(l)));
    }
    const float reg_beta = (float)(-tau * lambda), tau_f = (float)tau;

    /* 5. iterations (btv_l1_cuda.cpp:364-396) */
    for (int it = 0; it < iterations; ++it) {
        for (int k = 0; k < K; ++k) {
            remap_nearest(hr, (int)HH, (int)WW, C, bmap + 2 * k * hp, bmap + (2 * k + 1) * hp, a); /* a = M Ih */
            sr_model_sep_filter(a, (int)HH, (int)WW, C, kern, blur_kernel_size, b);               /* b = H M Ih */
            for (int y = 0; y < H; ++y)                                                           /* c = D H M Ih */
                for (int x = 0; x < W; ++x)
                    for (int ch = 0; ch < C; ++ch)
                        c[((size_t)y * W + x) * C + ch] = b[((size_t)y * s * WW + (size_t)x * s) * C + ch];
            for (size_t i = 0; i < lp * C; ++i) c[i] = diff_sign(src[(size_t)k * lp * C + i], c[i]);
            memset(a, 0, sizeof(float) * hp * C); /* a = Dt diff */
            for (int y = 0; y < H; ++y)
                for (int x = 0; x < W; ++x)
                    for (int ch = 0; ch < C; ++ch)
                        a[((size_t)y * s * WW + (size_t)x * s) * C + ch] = c[((size_t)y * W + x) * C + ch];
            sr_model_sep_filter(a, (int)HH, (int)WW, C, kern, blur_kernel_size, b); /* b = Ht Dt diff */
            remap_nearest(b, (int)HH, (int)WW, C, fmap + 2 * k * hp, fmap + (2 * k + 1) * hp, diff + (size_t)k * hp * C);
        }
        if (lambda > 0) {
            /* calcBtvRegularization: interior only, 0 elsewhere; the float4 diffSign zeroes the 4th channel */
            memset(reg, 0, sizeof(float) * hp * C);
            const int creg = C == 4 ? 3 : C;
            for (int y = ks; y < (int)HH - ks; ++y)
                for (int x = ks; x < (int)WW - ks; ++x)
                    for (int ch = 0; ch < creg; ++ch) {
                        const float v = hr[((size_t)y * WW + x) * C + ch];
                        float acc = 0.0f;
                        for (int m = 0, count = 0; m <= ks; ++m)
                            for (int l = ks; l + m >= 0; --l, ++count)
                                acc = acc + w[count] * (diff_sign(v, hr[((size_t)(y + m) * WW + x + l) * C + ch]) -
                                                        diff_sign(hr[((size_t)(y - m) * WW + x - l) * C + ch], v));
                        reg[((size_t)y * WW + x) * C + ch] = acc;
                    }
            for (size_t i = 0; i < hp * C; ++i) hr[i] = hr[i] * 1.0f + reg[i] * reg_beta + 0.0f; /* addWeighted */
        }
        for (int k = 0; k < K; ++k)
            for (size_t i = 0; i < hp * C; ++i) hr[i] = hr[i] * 1.0f + diff[(size_t)k * hp * C + i] * tau_f + 0.0f;
    }
    free(relF), free(relB), free(fmap), free(bmap), free(up), free(a), free(b), free(c), free(diff), free(reg);
    return 0;
}
