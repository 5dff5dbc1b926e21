/* brox_model.c -- C/OpenMP restatement of oracle/brox_model.py, operation for operation.
 * TEST INFRASTRUCTURE (see oracle/__init__.py).  Float only, built with -ffp-contract=off: every rounding is explicit,
 * fmaf() exactly where opencv_contrib_b200/csrc/brox.cu fuses.  Bit-identical to the numpy model (counters included)
 * and, with rsqrt mode 0 (correctly rounded), to the engine with aux_path 1.
 * Red-black SOR in place equals the kernels' ping-pong: a colour's update reads only the other colour. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <omp.h>

#define EPS2 1e-6f
enum { C_MIRRORED = 0, C_DEGENERATE, C_LEVELS, N_COUNTERS };

int brox_model_n_counters(void) { return N_COUNTERS; }
int brox_model_set_threads(int n) {
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
}

static int is_rounded_rsqrt(float x, float r) {
    /* r = 1/sqrt(x) to nearest: m_lo^2 x < 1 < m_hi^2 x for the midpoints m towards r's neighbours.  m^2 is exact in
     * double (2 x 25 bits) and fma(m^2, x, -1) rounds the exact m^2 x - 1 once, so its sign is exact.  No tie exists. */
    const double lo = 0.5 * ((double)r + (double)nextafterf(r, 0.0f));
    const double hi = 0.5 * ((double)r + (double)nextafterf(r, INFINITY));
    return fma(lo * lo, (double)x, -1.0) < 0.0 && fma(hi * hi, (double)x, -1.0) > 0.0;
}

/* 1/sqrt(x) correctly rounded (__frsqrt_rn) for positive finite x.  (float)(1.0 / sqrt((double)x)) rounds twice and can
 * misround, so the candidate is checked exactly and replaced by the neighbour that is. */
float brox_model_rsqrt_rn(float x) {
    float r = (float)(1.0 / sqrt((double)x));
    if (is_rounded_rsqrt(x, r)) return r;
    const float a = nextafterf(r, 0.0f), b = nextafterf(r, INFINITY);
    return is_rounded_rsqrt(x, a) ? a : b;
}

void brox_model_rsqrt_batch(const float *x, long n, float *r) {
#pragma omp parallel for schedule(static)
    for (long i = 0; i < n; ++i) r[i] = brox_model_rsqrt_rn(x[i]);
}

static int perturb_ulps(int level, int inner, uint32_t idx) {
    uint32_t h = idx * 2654435761u;
    h ^= (uint32_t)(level * 40503 + inner * 9973 + 1);
    h ^= h >> 15;
    h *= 2246822519u;
    h ^= h >> 13;
    return (int)(h % 5u) - 2;
}

static float data_rsqrt(float r2, int mode, int level, int inner, uint32_t idx) {
    float r = brox_model_rsqrt_rn(r2);
    if (mode == 1 && isfinite(r) && r > 1.17549435e-38f) {
        int32_t b;
        memcpy(&b, &r, 4);
        b += perturb_ulps(level, inner, idx);
        memcpy(&r, &b, 4);
    }
    return r;
}

static int mirror_filter(int i, int n) {
    if (i < 0) i = 1 - i;
    if (i >= n) i = n + n - i - 1;
    return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
}
static int mirror_tex(long i, int n) {
    const long p = 2L * n;
    i %= p;
    if (i < 0) i += p;
    return (int)(i >= n ? p - 1 - i : i);
}
static int mirror_load(int i, int n) {
    i = i > -i - 1 ? i : -i - 1;
    i = i < n - i + n - 1 ? i : n - i + n - 1;
    return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
}
static int clampi(int v, int a, int b) { return v < a ? a : (v > b ? b : v); }

static float tex_bilinear(const float *P, int h, int w, float xn, float yn, int *mirrored) {
    const float xb = fmaf(xn, (float)w, -0.5f), yb = fmaf(yn, (float)h, -0.5f);
    const float fx0 = floorf(xb), fy0 = floorf(yb);
    const float ax = xb - fx0, ay = yb - fy0;
    const float bx = 1.f - ax, by = 1.f - ay;
    const int x0 = (int)fminf(fmaxf(fx0, -1.0e6f), 1.0e6f), y0 = (int)fminf(fmaxf(fy0, -1.0e6f), 1.0e6f);
    if (mirrored) *mirrored = x0 < 0 || x0 + 1 >= w || y0 < 0 || y0 + 1 >= h;
    const int xa = mirror_tex(x0, w), xc = mirror_tex((long)x0 + 1, w);
    const int ya = mirror_tex(y0, h), yc = mirror_tex((long)y0 + 1, h);
    const float top = fmaf(bx, P[(size_t)ya * w + xa], ax * P[(size_t)ya * w + xc]);
    const float bot = fmaf(bx, P[(size_t)yc * w + xa], ax * P[(size_t)yc * w + xc]);
    return fmaf(by, top, ay * bot);
}

static float ss_line(const float *row, int sw, float xmin, float xmax, int ixmin, int ixmax, float fxmin, float cxmax) {
    const float w0 = (1.0f - xmin) + fxmin;
    float wsum = w0, sum = row[ixmin] * w0;
    int sp = ixmin + 1;
    for (int ix = ixmin + 1; ix < ixmax; ++ix) {
        sum = sum + row[sp < sw - 1 ? sp : sw - 1];
        sp++;
        wsum = wsum + 1.0f;
    }
    const float w1 = cxmax - xmax;
    sum = fmaf(w1, row[sp < sw - 1 ? sp : sw - 1], sum);
    wsum = wsum + w1;
    return sum / wsum;
}

static long supersample(const float *src, int sh, int sw, float *dst, int dh, int dw, float scale) {
    long deg = 0;
#pragma omp parallel for schedule(static) reduction(+ : deg)
    for (int iy = 0; iy < dh; ++iy) {
        for (int ix = 0; ix < dw; ++ix) {
            const float rw = (float)sw, rh = (float)sh, fx = (float)ix, fy = (float)iy;
            const float xBegin = fmaxf(fmaf(fx, scale, -scale), 0.0f), xEnd = fminf(fmaf(fx, scale, scale), rw - 1.0f);
            const float yBegin = fmaxf(fmaf(fy, scale, -scale), 0.0f), yEnd = fminf(fmaf(fy, scale, scale), rh - 1.0f);
            const float fxb = floorf(xBegin), cxe = ceilf(xEnd), fyb = floorf(yBegin), cye = ceilf(yEnd);
            const int iXBegin = (int)fxb, iXEnd = (int)cxe, iYBegin = (int)fyb, iYEnd = (int)cye;
            deg += iXEnd == iXBegin || iYEnd == iYBegin;
            int ry = iYBegin;
            const float w0 = (1.0f - yBegin) + fyb;
            float wsum = w0;
            float sum = ss_line(src + (size_t)ry * sw, sw, xBegin, xEnd, iXBegin, iXEnd, fxb, cxe) * w0;
            ry++;
            for (int yy = iYBegin + 1; yy < iYEnd; ++yy) {
                sum = sum + ss_line(src + (size_t)(ry < sh - 1 ? ry : sh - 1) * sw, sw, xBegin, xEnd, iXBegin, iXEnd, fxb, cxe);
                ry++;
                wsum = wsum + 1.0f;
            }
            const float w1 = cye - yEnd;
            sum = fmaf(w1, ss_line(src + (size_t)(ry < sh - 1 ? ry : sh - 1) * sw, sw, xBegin, xEnd, iXBegin, iXEnd, fxb, cxe),
                       sum);
            wsum = wsum + w1;
            dst[(size_t)iy * dw + ix] = sum / wsum;
        }
    }
    return deg;
}

/* {1,-8,0,8,-1}/12 with the reference's mirror rule; the products are exact, so fusing them cannot change a bit */
static void d5(const float *P, int h, int w, float *out, int along_x) {
#pragma omp parallel for schedule(static)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w; ++x) {
            static const float k[5] = {1.0f, -8.0f, 0.0f, 8.0f, -1.0f};
            float sum = 0.0f;
            for (int m = 0; m < 5; ++m) {
                const float v = along_x ? P[(size_t)y * w + mirror_filter(x + m - 2, w)]
                                        : P[(size_t)mirror_filter(y + m - 2, h) * w + x];
                sum = sum + v * k[m];
            }
            out[(size_t)y * w + x] = sum * (1.0f / 12.0f);
        }
    }
}

static float bicubic_coeff(float x_) {
    const float x = fabsf(x_);
    if (x <= 1.0f) return fmaf(x * x, fmaf(x, 1.5f, -2.5f), 1.0f);
    if (x < 2.0f) return fmaf(x, fmaf(x, fmaf(x, -0.5f, 2.5f), -4.0f), 2.0f);
    return 0.0f;
}

static void prolong(const float *src, int sh, int sw, float *dst, int dh, int dw, float scale, float mul) {
#pragma omp parallel for schedule(static)
    for (int iy = 0; iy < dh; ++iy) {
        for (int ix = 0; ix < dw; ++ix) {
            const float rw = (float)sw, rh = (float)sh, fx = (float)ix, fy = (float)iy;
            const float xmin = fmaxf(ceilf(fmaf(fx, scale, -2.0f)), 0.0f), xmax = fminf(floorf(fmaf(fx, scale, 2.0f)), rw - 1.0f);
            const float ymin = fmaxf(ceilf(fmaf(fy, scale, -2.0f)), 0.0f), ymax = fminf(floorf(fmaf(fy, scale, 2.0f)), rh - 1.0f);
            float sum = 0.0f, wsum = 0.0f;
            for (float cy = ymin; cy <= ymax; cy = cy + 1.0f) {
                for (float cx = xmin; cx <= xmax; cx = cx + 1.0f) {
                    float wx = bicubic_coeff(fmaf(fx, scale, -cx));
                    const float wy = bicubic_coeff(fmaf(fy, scale, -cy));
                    wx = wx * wy;
                    sum = fmaf(wx, src[(size_t)(int)cy * sw + (int)cx], sum);
                    wsum = wsum + wx;
                }
            }
            const float r = (wsum == 0.0f) ? 0.f : sum / wsum;
            dst[(size_t)iy * dw + ix] = r * mul;
        }
    }
}

static float diffusivity(float u_x, float v_x, float u_y, float v_y) {
    float s = fmaf(u_x, u_x, v_x * v_x);
    s = fmaf(u_y, u_y, s);
    s = fmaf(v_y, v_y, s);
    return 0.5f / sqrtf(s + EPS2);
}

typedef struct {
    int h, w;
    const float *u, *v;
    float *du, *dv;
    const float *W[8]; /* Iz, Ix, Ixz, Ixy, Ixx, Iy, Iyz, Iyy */
    float *sx, *sy, *inv_u, *inv_v, *num_dudv, *num_u, *num_v;
} Level;

#define AT(p, y, x) (p)[(size_t)(y) * L->w + (x)]
static float brox_sx(const Level *L, int j, int i) {
    const int h = L->h, w = L->w;
    const int i0 = mirror_load(i, w), im = mirror_load(i - 1, w);
    const int j0 = mirror_load(j, h), jp = mirror_load(j + 1, h), jm = mirror_load(j - 1, h);
    const float *u = L->u, *du = L->du, *v = L->v, *dv = L->dv;
    const float u_x = AT(u, j0, i0) + AT(du, j0, i0) - AT(u, j0, im) - AT(du, j0, im);
    const float v_x = AT(v, j0, i0) + AT(dv, j0, i0) - AT(v, j0, im) - AT(dv, j0, im);
    const float u_y = 0.25f * (AT(u, jp, i0) + AT(du, jp, i0) + AT(u, jp, im) + AT(du, jp, im) - AT(u, jm, i0) -
                               AT(du, jm, i0) - AT(u, jm, im) - AT(du, jm, im));
    const float v_y = 0.25f * (AT(v, jp, i0) + AT(dv, jp, i0) + AT(v, jp, im) + AT(dv, jp, im) - AT(v, jm, i0) -
                               AT(dv, jm, i0) - AT(v, jm, im) - AT(dv, jm, im));
    return diffusivity(u_x, v_x, u_y, v_y);
}
static float brox_sy(const Level *L, int j, int i) {
    const int h = L->h, w = L->w;
    const int i0 = mirror_load(i, w), ip = mirror_load(i + 1, w), im = mirror_load(i - 1, w);
    const int j0 = mirror_load(j, h), jm = mirror_load(j - 1, h);
    const float *u = L->u, *du = L->du, *v = L->v, *dv = L->dv;
    const float u_y = AT(u, j0, i0) + AT(du, j0, i0) - AT(u, jm, i0) - AT(du, jm, i0);
    const float v_y = AT(v, j0, i0) + AT(dv, j0, i0) - AT(v, jm, i0) - AT(dv, jm, i0);
    const float u_x = 0.25f * (AT(u, j0, ip) + AT(u, jm, ip) + AT(du, j0, ip) + AT(du, jm, ip) - AT(u, j0, im) -
                               AT(u, jm, im) - AT(du, j0, im) - AT(du, jm, im));
    const float v_x = 0.25f * (AT(v, j0, ip) + AT(v, jm, ip) + AT(dv, j0, ip) + AT(dv, jm, ip) - AT(v, j0, im) -
                               AT(v, jm, im) - AT(dv, j0, im) - AT(dv, jm, im));
    return diffusivity(u_x, v_x, u_y, v_y);
}

static void prepare(Level *L, float alpha, float gamma, int mode, int level, int inner) {
    const int h = L->h, w = L->w;
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j)
        for (int i = 0; i < w; ++i) {
            AT(L->sx, j, i) = i == 0 ? 0.f : brox_sx(L, j, i);
            AT(L->sy, j, i) = j == 0 ? 0.f : brox_sy(L, j, i);
        }
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j)
        for (int i = 0; i < w; ++i) {
            const size_t p = (size_t)j * w + i;
            const float du = L->du[p], dv = L->dv[p];
            const float Iz = L->W[0][p], Ix = L->W[1][p], Ixz = L->W[2][p], Ixy = L->W[3][p];
            const float Ixx = L->W[4][p], Iy = L->W[5][p], Iyz = L->W[6][p], Iyy = L->W[7][p];
            const float q0 = fmaf(dv, Iy, fmaf(du, Ix, Iz));
            const float q1 = fmaf(dv, Ixy, fmaf(du, Ixx, Ixz));
            const float q2 = fmaf(dv, Iyy, fmaf(du, Ixy, Iyz));
            const float r2 = fmaf(q0, q0, gamma * fmaf(q1, q1, q2 * q2)) + EPS2;
            float data = 0.5f * data_rsqrt(r2, mode, level, inner, (uint32_t)p);
            data = data / alpha;
            const float sx = L->sx[p], sxr = i < w - 1 ? L->sx[p + 1] : 0.f;
            const float sy = L->sy[p], syu = j < h - 1 ? L->sy[p + w] : 0.f;
            L->num_dudv[p] = data * fmaf(Ix, Iy, (gamma * Ixy) * (Ixx + Iyy));
            L->num_u[p] = data * fmaf(Ix, Iz, gamma * fmaf(Ixx, Ixz, Ixy * Iyz));
            L->num_v[p] = data * fmaf(Iy, Iz, gamma * fmaf(Ixy, Ixz, Iyy * Iyz));
            const float den_u = fmaf(Ix, Ix, gamma * fmaf(Ixy, Ixy, Ixx * Ixx));
            const float den_v = fmaf(Iy, Iy, gamma * fmaf(Ixy, Ixy, Iyy * Iyy));
            const float dsum = ((sx + sxr) + sy) + syu;
            L->inv_u[p] = 1.0f / fmaf(data, den_u, dsum);
            L->inv_v[p] = 1.0f / fmaf(data, den_v, dsum);
        }
}

static void sor_colour(Level *L, int colour) {
    const int h = L->h, w = L->w;
    const float omega = 1.99f, omo = 1.0f - omega;
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        for (int i = (j + colour) & 1; i < w; i += 2) {
            const int ir = i < w - 1 ? i + 1 : i, il = i > 0 ? i - 1 : i;
            const int ju = j < h - 1 ? j + 1 : j, jd = j > 0 ? j - 1 : j;
            const size_t p = (size_t)j * w + i;
            const float s_l = L->sx[p], s_d = L->sy[p];
            const float s_r = i < w - 1 ? AT(L->sx, j, ir) : 0.0f, s_u = j < h - 1 ? AT(L->sy, ju, i) : 0.0f;
            const float ssum = ((s_l + s_r) + s_u) + s_d;
            const float usum = L->u[p] * ssum, vsum = L->v[p] * ssum;
            const float w_u = omega * L->inv_u[p], w_v = omega * L->inv_v[p];
#define UU(y, x) (AT(L->u, y, x) + AT(L->du, y, x))
#define VV(y, x) (AT(L->v, y, x) + AT(L->dv, y, x))
            float t = s_l * UU(j, il);
            t = fmaf(s_u, UU(ju, i), t);
            t = fmaf(s_r, UU(j, ir), t);
            t = fmaf(s_d, UU(jd, i), t);
            t = t - usum;
            t = t - L->num_u[p];
            t = fmaf(-L->num_dudv[p], L->dv[p], t);
            const float du = fmaf(w_u, t, omo * L->du[p]);
            t = s_l * VV(j, il);
            t = fmaf(s_u, VV(ju, i), t);
            t = fmaf(s_r, VV(j, ir), t);
            t = fmaf(s_d, VV(jd, i), t);
            t = t - vsum;
            t = t - L->num_v[p];
            t = fmaf(-L->num_dudv[p], du, t);
            L->dv[p] = fmaf(w_v, t, omo * L->dv[p]);
            L->du[p] = du;
#undef UU
#undef VV
        }
    }
}
#undef AT

/* pyramid sizes: ceilf(src * scale) with a cumulative float scale, stop at <= 15 px or the level cap (NB:730-785) */
static int pyramid_sizes(int h, int w, float sf, int outer, int *hs, int *ws, int cap) {
    int n = 1, pw = w, ph = h;
    float scale = 1.0f * sf;
    hs[0] = h;
    ws[0] = w;
    while (pw > 15 && ph > 15 && n < outer && n < cap) {
        ws[n] = (int)ceilf((float)w * scale);
        hs[n] = (int)ceilf((float)h * scale);
        pw = ws[n];
        ph = hs[n];
        scale = scale * sf;
        ++n;
    }
    return n;
}

/* Returns 0, -1 on allocation failure, -2 on bad arguments. */
int brox_model_calc(const float *I0, const float *I1, int h, int w, float alpha, float gamma, float scale_factor, int inner,
                    int outer, int solver, int rsqrt_mode, float *flow, long long *counters) {
    enum { CAP = 256 };
    if (h <= 0 || w <= 0 || inner <= 0 || outer <= 0 || solver <= 0 || rsqrt_mode < 0 || rsqrt_mode > 1) return -2;
    int hs[CAP], ws[CAP];
    const int nl = pyramid_sizes(h, w, scale_factor, outer, hs, ws, CAP);
    for (int k = 0; k < N_COUNTERS; ++k) counters[k] = 0;
    const size_t N = (size_t)h * w;
    float *pyr0[CAP], *pyr1[CAP];
    float *buf = malloc(sizeof(float) * N * 30);
    int ok = buf != NULL;
    for (int l = 0; l < nl; ++l) {
        pyr0[l] = malloc(sizeof(float) * (size_t)hs[l] * ws[l]);
        pyr1[l] = malloc(sizeof(float) * (size_t)hs[l] * ws[l]);
        ok = ok && pyr0[l] && pyr1[l];
    }
    if (!ok) {
        for (int l = 0; l < nl; ++l) { free(pyr0[l]); free(pyr1[l]); }
        free(buf);
        return -1;
    }
    memcpy(pyr0[0], I0, sizeof(float) * N);
    memcpy(pyr1[0], I1, sizeof(float) * N);
    const float inv_sf = 1.0f / scale_factor;
    for (int l = 1; l < nl; ++l) {
        counters[C_DEGENERATE] += supersample(pyr0[l - 1], hs[l - 1], ws[l - 1], pyr0[l], hs[l], ws[l], inv_sf);
        supersample(pyr1[l - 1], hs[l - 1], ws[l - 1], pyr1[l], hs[l], ws[l], inv_sf);
    }
    float *pl[30];
    for (int k = 0; k < 30; ++k) pl[k] = buf + N * k;
    float *u = pl[0], *v = pl[1], *un = pl[2], *vn = pl[3];
    float *Ix0 = pl[4], *Iy0 = pl[5], *Ix = pl[6], *Iy = pl[7], *Ixx = pl[8], *Iyy = pl[9], *Ixy = pl[10];
    memset(u, 0, sizeof(float) * (size_t)hs[nl - 1] * ws[nl - 1]);
    memset(v, 0, sizeof(float) * (size_t)hs[nl - 1] * ws[nl - 1]);
    for (int l = nl - 1; l >= 0; --l) {
        const int lh = hs[l], lw = ws[l];
        const size_t n = (size_t)lh * lw;
        Level L = {lh, lw, u, v, pl[11], pl[12], {pl[13], pl[14], pl[15], pl[16], pl[17], pl[18], pl[19], pl[20]},
                   pl[21], pl[22], pl[23], pl[24], pl[25], pl[26], pl[27]};
        memset(L.du, 0, sizeof(float) * n);
        memset(L.dv, 0, sizeof(float) * n);
        d5(pyr0[l], lh, lw, Ix0, 1);
        d5(pyr0[l], lh, lw, Iy0, 0);
        d5(pyr1[l], lh, lw, Ix, 1);
        d5(pyr1[l], lh, lw, Iy, 0);
        d5(Ix, lh, lw, Ixx, 1);
        d5(Iy, lh, lw, Iyy, 0);
        d5(Iy, lh, lw, Ixy, 1);
        long mirrored = 0;
        float **W = (float **)L.W;
#pragma omp parallel for schedule(static) reduction(+ : mirrored)
        for (int jg = 0; jg < lh; ++jg) {
            for (int ig = 0; ig < lw; ++ig) {
                const size_t p = (size_t)jg * lw + ig;
                float x = (float)ig + 0.5f, y = (float)jg + 0.5f;
                const float wx = (x + u[p]) / (float)lw, wy = (y + v[p]) / (float)lh;
                x = x / (float)lw;
                y = y / (float)lh;
                int mir = 0;
                const float ix = tex_bilinear(Ix, lh, lw, wx, wy, &mir);
                const float iy = tex_bilinear(Iy, lh, lw, wx, wy, NULL);
                mirrored += mir;
                W[0][p] = tex_bilinear(pyr1[l], lh, lw, wx, wy, NULL) - tex_bilinear(pyr0[l], lh, lw, x, y, NULL);
                W[1][p] = ix;
                W[2][p] = ix - tex_bilinear(Ix0, lh, lw, x, y, NULL);
                W[3][p] = tex_bilinear(Ixy, lh, lw, wx, wy, NULL);
                W[4][p] = tex_bilinear(Ixx, lh, lw, wx, wy, NULL);
                W[5][p] = iy;
                W[6][p] = iy - tex_bilinear(Iy0, lh, lw, x, y, NULL);
                W[7][p] = tex_bilinear(Iyy, lh, lw, wx, wy, NULL);
            }
        }
        counters[C_MIRRORED] += mirrored;
        for (int it = 0; it < inner; ++it) {
            prepare(&L, alpha, gamma, rsqrt_mode, l, it);
            for (int s = 0; s < solver; ++s) {
                sor_colour(&L, 0);
                sor_colour(&L, 1);
            }
        }
        for (size_t p = 0; p < n; ++p) {
            u[p] = u[p] + L.du[p];
            v[p] = v[p] + L.dv[p];
        }
        counters[C_LEVELS] += 1;
        if (l > 0) {
            prolong(u, lh, lw, un, hs[l - 1], ws[l - 1], 1.0f / inv_sf, inv_sf);
            prolong(v, lh, lw, vn, hs[l - 1], ws[l - 1], 1.0f / inv_sf, inv_sf);
            float *t = u; u = un; un = t;
            t = v; v = vn; vn = t;
        }
    }
    for (size_t p = 0; p < N; ++p) {
        flow[2 * p] = u[p];
        flow[2 * p + 1] = v[p];
    }
    for (int l = 0; l < nl; ++l) { free(pyr0[l]); free(pyr1[l]); }
    free(buf);
    return 0;
}
