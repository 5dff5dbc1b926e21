// optflowgf.cu -- the video module's Farneback flow (cv::calcOpticalFlowFarneback, cv::FarnebackOpticalFlow) for
// sm_90a, bit for bit equal to cv2 4.x's portable CPU path (setUseOptimized(false), IPP off).  oracle/optflowgf_model.py
// states every rounding and summation order; DESIGN §4.14 gives the argument.  Built with -fmad=false, so each float and
// double expression rounds once per operation, in the order written, as the model does.
//
// Per call: both frames converted to float (1 launch, outside the graph), the caller's flow split (1, with
// OPTFLOW_USE_INITIAL_FLOW); inside the handle's CUDA graph, per level from the coarsest: the full-size row blur (1), the
// level images by the column blur fused with the centre-aligned resize (1), the polynomial expansion of both frames
// (vertical 1, horizontal 1), the initial or prolonged flow (1), updateMatrices (1), then per iteration the window solve
// (box: a vertical and a horizontal running-sum pass; gaussian: vertical and horizontal float sums) and, except after the
// last, updateMatrices; last the merge into the caller's flow (1, outside the graph).
//
// The box window's double running sums are sequential by definition: its vertical pass runs one thread per column and
// plane, its horizontal pass one thread per row carrying the five sums, over vertical sums stored transposed so that both
// passes touch memory coalesced.  Both are latency-bound; several handles on several streams (b2f_batch) recover
// throughput.  A handle may be called on any stream: a call on another stream than the previous call waits for it.
//
// Kernel classes: 0 blur and level images, 1 polynomial expansion, 2 updateMatrices, 3 window solve, 4 flow I/O.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <new>

#include "common.cuh"

namespace b2f {
namespace {

enum { CLS_LEVEL = 0, CLS_POLY = 1, CLS_UPDATE = 2, CLS_SOLVE = 3, CLS_IO = 4 };
constexpr int GF_MAX_BLUR = 255;  // level-blur taps: ksize grows like 2.5 / pyrScale^k, 255 covers frames up to ~6000 px
constexpr int GF_MAX_POLY_N = B2F_OPTFLOWGF_MAX_POLY_N;
constexpr int GF_MAX_WIN = B2F_OPTFLOWGF_MAX_WIN_SIZE;
constexpr int BS = 256;

struct BlurTaps {
    float k[GF_MAX_BLUR];
    int ksize;
};
struct PolyTaps {
    float g[2 * GF_MAX_POLY_N + 1], xg[2 * GF_MAX_POLY_N + 1], xxg[2 * GF_MAX_POLY_N + 1];
    double ig11, ig03, ig33, ig55;
    int n;
};
struct WinTaps {
    float k[GF_MAX_WIN / 2 + 1];
    int m;
};

__device__ __forceinline__ int reflect101(int p, int n) {
    if (n == 1) return 0;
    while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * (n - 1) - p;
    return p;
}

// ---------------------------------------------------------------------------------------------------------------
// Level images: GaussianBlur of the full-size float frame, then resize INTER_LINEAR to the level size
// ---------------------------------------------------------------------------------------------------------------

// resize INTER_LINEAR source taps of one destination index: horizontally (clamp) a tap outside the source moves to the
// edge with fraction 0, vertically only the indices clamp
__device__ __forceinline__ void linear_tap(int d, double scale, int n_src, bool clamp, int &i0, int &i1, float &f) {
    f = static_cast<float>((d + 0.5) * scale - 0.5);
    const float fl = floorf(f);
    int s = static_cast<int>(fl);
    f = f - static_cast<float>(s);
    if (clamp && s < 0) { s = 0; f = 0.f; }
    if (clamp && s >= n_src - 1) { s = n_src - 1; f = 0.f; }
    i0 = min(max(s, 0), n_src - 1);
    i1 = min(max(s + 1, 0), n_src - 1);
}

// the row pass: kc x + k1 (l1 + r1) + k2 (l2 + r2) for ksize <= 5, the sequential k0 x0 + k1 x1 + ... above.  Every
// column of the level reads two blurred columns (x0, x1) of the frame; when the level has fewer than half the frame's
// columns (`compact`), only those are computed, column 2 dx + i of T holding tap i of level column dx.  Every row is
// computed: the column blur spans about 2.5 / scale rows around taps 1 / scale apart, so it reads them all.
__global__ void k_gf_blur_rows(Plane F0, Plane F1, Plane T0, Plane T1, int cols, int tcols, int compact, double sx,
                               BlurTaps t) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (j >= tcols) return;
    int x = j;
    if (compact) {
        int x0, x1;
        float f;
        linear_tap(j >> 1, sx, cols, true, x0, x1, f);
        x = (j & 1) ? x1 : x0;
    }
    const float *s = (blockIdx.z ? F1 : F0).row(y);
    const int r = t.ksize / 2;
    float acc;
    if (t.ksize <= 5) {
        acc = t.k[r] * s[x];
        for (int i = 1; i <= r; ++i) acc = acc + t.k[r + i] * (s[reflect101(x - i, cols)] + s[reflect101(x + i, cols)]);
    } else {
        acc = t.k[0] * s[reflect101(x - r, cols)];
        for (int i = 1; i < t.ksize; ++i) acc = acc + t.k[i] * s[reflect101(x - r + i, cols)];
    }
    (blockIdx.z ? T1 : T0).at(y, j) = acc;
}

// the column pass at one pixel: kc x + sum k_i (up_i + down_i)
__device__ __forceinline__ float blur_col(const Plane &T, int y, int x, int rows, const BlurTaps &t) {
    const int r = t.ksize / 2;
    float acc = t.k[r] * T.at(y, x);
    for (int i = 1; i <= r; ++i) acc = acc + t.k[r + i] * (T.at(reflect101(y - i, rows), x) + T.at(reflect101(y + i, rows), x));
    return acc;
}

// mode 0: same size (copy), 1: resize INTER_LINEAR, 2: an exact 2x downscale (OpenCV's fast INTER_AREA)
__global__ void k_gf_level(Plane T0, Plane T1, Plane I0, Plane I1, int rows, int cols, int lcols, int mode, int compact,
                           double sx, double sy, BlurTaps t) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= lcols) return;
    const Plane &T = blockIdx.z ? T1 : T0;
    float out;
    if (mode == 0) {
        out = blur_col(T, y, x, rows, t);
    } else if (mode == 2) {
        const float a = blur_col(T, 2 * y, 2 * x, rows, t), b = blur_col(T, 2 * y, 2 * x + 1, rows, t);
        const float c = blur_col(T, 2 * y + 1, 2 * x, rows, t), d = blur_col(T, 2 * y + 1, 2 * x + 1, rows, t);
        if (x < lcols - lcols % 4) {
            out = ((a + b) + (c + d)) * 0.25f;  // the 4-wide vector path
        } else {
            float s = 0.f;
            s = s + (((a + b) + c) + d);
            out = s * 0.25f;
        }
    } else {
        int x0, x1, y0, y1;
        float fx, fy;
        linear_tap(x, sx, cols, true, x0, x1, fx);
        if (compact) {
            x0 = 2 * x;
            x1 = 2 * x + 1;
        }
        linear_tap(y, sy, rows, false, y0, y1, fy);
        const float t0 = blur_col(T, y0, x0, rows, t) * (1.f - fx) + blur_col(T, y0, x1, rows, t) * fx;
        const float t1 = blur_col(T, y1, x0, rows, t) * (1.f - fx) + blur_col(T, y1, x1, rows, t) * fx;
        out = t0 * (1.f - fy) + t1 * fy;
    }
    (blockIdx.z ? I1 : I0).at(y, x) = out;
}

// ---------------------------------------------------------------------------------------------------------------
// Polynomial expansion (FarnebackPolyExp), both frames per launch
// ---------------------------------------------------------------------------------------------------------------
struct Planes5 {
    Plane p[5];
};
struct Planes3x2 {
    Plane p[6];
};

__global__ void k_gf_poly_v(Plane I0, Plane I1, Planes3x2 out, int rows, int cols, PolyTaps t) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    const Plane &S = blockIdx.z ? I1 : I0;
    const int n = t.n;
    float r0 = S.at(y, x) * t.g[n], r1 = 0.f, r2 = 0.f;
    for (int k = 1; k <= n; ++k) {
        const float s0 = S.at(max(y - k, 0), x), s1 = S.at(min(y + k, rows - 1), x);
        const float p = s0 + s1;
        r0 = r0 + t.g[n + k] * p;
        r1 = r1 + t.xg[n + k] * (s1 - s0);
        r2 = r2 + t.xxg[n + k] * p;
    }
    const int o = blockIdx.z * 3;
    out.p[o].at(y, x) = r0;
    out.p[o + 1].at(y, x) = r1;
    out.p[o + 2].at(y, x) = r2;
}

__global__ void k_gf_poly_h(Planes3x2 in, Planes5 R0, Planes5 R1, int cols, PolyTaps t) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    const int o = blockIdx.z * 3;
    const float *a = in.p[o].row(y), *b = in.p[o + 1].row(y), *c = in.p[o + 2].row(y);
    const int n = t.n;
    const float g0 = t.g[n];
    double b1 = static_cast<double>(a[x] * g0), b2 = 0, b3 = static_cast<double>(b[x] * g0), b4 = 0,
           b5 = static_cast<double>(c[x] * g0), b6 = 0;
    for (int k = 1; k <= n; ++k) {
        const int R = min(x + k, cols - 1), L = max(x - k, 0);
        const double tg = static_cast<double>(a[R] + a[L]);
        const float gk = t.g[n + k];
        b1 = b1 + tg * static_cast<double>(gk);
        b4 = b4 + tg * static_cast<double>(t.xxg[n + k]);
        b2 = b2 + static_cast<double>((a[R] - a[L]) * t.xg[n + k]);
        b3 = b3 + static_cast<double>((b[R] + b[L]) * gk);
        b6 = b6 + static_cast<double>((b[R] - b[L]) * t.xg[n + k]);
        b5 = b5 + static_cast<double>((c[R] + c[L]) * gk);
    }
    const Planes5 &D = blockIdx.z ? R1 : R0;
    D.p[1].at(y, x) = static_cast<float>(b2 * t.ig11);
    D.p[0].at(y, x) = static_cast<float>(b3 * t.ig11);
    D.p[3].at(y, x) = static_cast<float>(b1 * t.ig03 + b4 * t.ig33);
    D.p[2].at(y, x) = static_cast<float>(b1 * t.ig03 + b5 * t.ig33);
    D.p[4].at(y, x) = static_cast<float>(b6 * t.ig55);
}

// ---------------------------------------------------------------------------------------------------------------
// FarnebackUpdateMatrices over the whole field
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float border_w(int i) {
    return i == 0 ? 0.14f : i == 1 ? 0.14f : 0.4472f;
}

__global__ void k_gf_update(Planes5 R0, Planes5 R1, Plane U, Plane V, Planes5 M, int rows, int cols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    const float dx = U.at(y, x), dy = V.at(y, x);
    float fx = static_cast<float>(x) + dx, fy = static_cast<float>(y) + dy;
    const float x1f = floorf(fx), y1f = floorf(fy);
    float r2, r3, r4, r5, r6;
    const float q0 = R0.p[0].at(y, x), q1 = R0.p[1].at(y, x), q2 = R0.p[2].at(y, x), q3 = R0.p[3].at(y, x),
                q4 = R0.p[4].at(y, x);
    if (x1f >= 0.f && x1f < static_cast<float>(cols - 1) && y1f >= 0.f && y1f < static_cast<float>(rows - 1)) {
        const int x1 = static_cast<int>(x1f), y1 = static_cast<int>(y1f);
        fx = fx - x1f;
        fy = fy - y1f;
        const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
        float r[5];
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            const Plane &P = R1.p[c];
            r[c] = ((a00 * P.at(y1, x1) + a01 * P.at(y1, x1 + 1)) + a10 * P.at(y1 + 1, x1)) + a11 * P.at(y1 + 1, x1 + 1);
        }
        r2 = r[0];
        r3 = r[1];
        r4 = (q2 + r[2]) * 0.5f;
        r5 = (q3 + r[3]) * 0.5f;
        r6 = (q4 + r[4]) * 0.25f;
    } else {
        r2 = r3 = 0.f;
        r4 = q2;
        r5 = q3;
        r6 = q4 * 0.5f;
    }
    r2 = (q0 - r2) * 0.5f;
    r3 = (q1 - r3) * 0.5f;
    r2 = r2 + (r4 * dy + r6 * dx);
    r3 = r3 + (r6 * dy + r5 * dx);
    // cv2's (unsigned)(x - 5) >= (unsigned)(width - 10)
    if ((unsigned)(x - 5) >= (unsigned)(cols - 10) || (unsigned)(y - 5) >= (unsigned)(rows - 10)) {
        const float s = (((x < 5 ? border_w(x) : 1.f) * (x >= cols - 5 ? border_w(cols - x - 1) : 1.f)) *
                         (y < 5 ? border_w(y) : 1.f)) *
                        (y >= rows - 5 ? border_w(rows - y - 1) : 1.f);
        r2 = r2 * s;
        r3 = r3 * s;
        r4 = r4 * s;
        r5 = r5 * s;
        r6 = r6 * s;
    }
    M.p[0].at(y, x) = r4 * r4 + r6 * r6;
    M.p[1].at(y, x) = (r4 + r5) * r6;
    M.p[2].at(y, x) = r5 * r5 + r6 * r6;
    M.p[3].at(y, x) = r4 * r2 + r6 * r3;
    M.p[4].at(y, x) = r6 * r2 + r5 * r3;
}

// ---------------------------------------------------------------------------------------------------------------
// Window solves
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void solve2(double g11, double g12, double g22, double h1, double h2, float &u, float &v) {
    const double idet = 1. / (g11 * g22 - g12 * g12 + 1e-3);
    u = static_cast<float>((g11 * h2 - g12 * h1) * idet);
    v = static_cast<float>((g22 * h1 - g12 * h2) * idet);
}

// box, vertical: one thread per (column, plane), a sequential double running sum down the rows.  The sums are stored
// transposed (plane c, column x, row y at vs[c * cstride + x * rpitch + y]) so that the horizontal pass, one thread per
// row, reads them coalesced; each 32-row block goes through shared memory so that these writes are coalesced too.
constexpr int BOX_TILE = 32;
__global__ void __launch_bounds__(BOX_TILE) k_gf_box_v(Planes5 M, double *vs, size_t cstride, size_t rpitch, int rows,
                                                      int cols, int m) {
    __shared__ double tile[BOX_TILE][BOX_TILE + 1];
    const int tid = threadIdx.x, x0 = blockIdx.x * BOX_TILE, x = x0 + tid, c = blockIdx.y;
    const Plane &P = M.p[c];
    const bool live = x < cols;
    double s = 0;
    if (live) {
        s = static_cast<double>(P.at(0, x) * static_cast<float>(m + 2));
        for (int y = 1; y < m; ++y) s = s + static_cast<double>(P.at(min(y, rows - 1), x));
    }
    double *o = vs + (size_t)c * cstride;
    for (int y0 = 0; y0 < rows; y0 += BOX_TILE) {
        const int n = min(BOX_TILE, rows - y0);
        for (int i = 0; i < n; ++i) {
            const int y = y0 + i;
            if (live) s = s + static_cast<double>(P.at(min(y + m, rows - 1), x) - P.at(max(y - m - 1, 0), x));
            tile[tid][i] = s;
        }
        __syncthreads();
        if (tid < n)
            for (int i = 0; i < BOX_TILE && x0 + i < cols; ++i) o[(size_t)(x0 + i) * rpitch + y0 + tid] = tile[i][tid];
        __syncthreads();
    }
}

// box, horizontal: one thread per row carries the five sums along it and writes the flow
__global__ void k_gf_box_h(const double *vs, size_t cstride, size_t rpitch, Plane U, Plane V, int rows, int cols, int m,
                           double scale) {
    const int y = blockIdx.x * blockDim.x + threadIdx.x;
    if (y >= rows) return;
    const double *r = vs + y;
    double g[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        g[c] = r[c * cstride] * static_cast<double>(m + 2);
        for (int x = 1; x < m; ++x) g[c] = g[c] + r[c * cstride + (size_t)min(x, cols - 1) * rpitch];
    }
    for (int x = 0; x < cols; ++x) {
        const size_t a = (size_t)min(x + m, cols - 1) * rpitch, b = (size_t)max(x - m - 1, 0) * rpitch;
        double sc[5];
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            g[c] = g[c] + (r[c * cstride + a] - r[c * cstride + b]);
            sc[c] = g[c] * scale;
        }
        float u, v;
        solve2(sc[0], sc[1], sc[2], sc[3], sc[4], u, v);
        U.at(y, x) = u;
        V.at(y, x) = v;
    }
}

// gaussian, vertical: float sums k0 M + sum k_i (down_i + up_i), replicated rows
__global__ void k_gf_gauss_v(Planes5 M, Planes5 G, int rows, int cols, WinTaps t) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, c = blockIdx.z;
    if (x >= cols) return;
    const Plane &P = M.p[c];
    float s = P.at(y, x) * t.k[0];
    for (int i = 1; i <= t.m; ++i) s = s + (P.at(min(y + i, rows - 1), x) + P.at(max(y - i, 0), x)) * t.k[i];
    G.p[c].at(y, x) = s;
}

// gaussian, horizontal, then the solve in double on the float sums
__global__ void k_gf_gauss_h(Planes5 G, Plane U, Plane V, int cols, WinTaps t) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    double h[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        const float *r = G.p[c].row(y);
        float s = r[x] * t.k[0];
        for (int i = 1; i <= t.m; ++i) s = s + t.k[i] * (r[max(x - i, 0)] + r[min(x + i, cols - 1)]);
        h[c] = static_cast<double>(s);
    }
    float u, v;
    solve2(h[0], h[1], h[2], h[3], h[4], u, v);
    U.at(y, x) = u;
    V.at(y, x) = v;
}

// ---------------------------------------------------------------------------------------------------------------
// Flow between levels
// ---------------------------------------------------------------------------------------------------------------

// Mat *= s on a float field: convertTo rounds float(x * float(s)) + 0.f
__device__ __forceinline__ float scale_val(float v, float s) { return v * s + 0.f; }

// prolongation: resize INTER_LINEAR of the 2-channel flow from the coarser level (never smaller, since pyrScale < 1, so
// resize's exact-half area rule cannot apply; mode 0 is an equal size, mode 1 the resize), then *= 1/pyrScale
__global__ void k_gf_prolong(Plane PU, Plane PV, Plane U, Plane V, int prows, int pcols, int rows, int cols, int mode,
                             double sx, double sy, float mul) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    const Plane &S = blockIdx.z ? PV : PU;
    float out;
    if (mode == 0) {
        out = S.at(y, x);
    } else {
        int x0, x1, y0, y1;
        float fx, fy;
        linear_tap(x, sx, pcols, true, x0, x1, fx);
        linear_tap(y, sy, prows, false, y0, y1, fy);
        const float t0 = S.at(y0, x0) * (1.f - fx) + S.at(y0, x1) * fx;
        const float t1 = S.at(y1, x0) * (1.f - fx) + S.at(y1, x1) * fx;
        out = t0 * (1.f - fy) + t1 * fy;
    }
    (blockIdx.z ? V : U).at(y, x) = scale_val(out, mul);
}

// computeResizeAreaTab for one destination index: source range [s1, s2) of weight 1/cw plus partial ends
struct AreaAxis {
    int lo, s1, s2, hi;  // lo = s1 - 1 when a leading partial tap exists, else -1; hi = s2 when a trailing one exists
    float wlo, wmid, whi;
};
__device__ __forceinline__ AreaAxis area_axis(int d, double scale, int n_src) {
    const double f1 = d * scale, f2 = f1 + scale;
    const double cw = fmin(scale, n_src - f1);
    int s1 = static_cast<int>(ceil(f1)), s2 = static_cast<int>(floor(f2));
    s2 = min(s2, n_src - 1);
    s1 = min(s1, s2);
    AreaAxis a;
    a.s1 = s1;
    a.s2 = s2;
    a.lo = s1 - f1 > 1e-3 ? s1 - 1 : -1;
    a.wlo = static_cast<float>((s1 - f1) / cw);
    a.wmid = static_cast<float>(1.0 / cw);
    a.hi = f2 - s2 > 1e-3 ? s2 : -1;
    a.whi = static_cast<float>(fmin(fmin(f2 - s2, 1.0), cw) / cw);
    return a;
}

// the caller's flow to the coarsest level: resize INTER_AREA (integer factors: the fast block sum), then *= scale
__global__ void k_gf_area(Plane SU, Plane SV, Plane U, Plane V, int srows, int scols, int rows, int cols, int ix, int iy,
                          double sx, double sy, float mul, int apply_mul) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    const Plane &S = blockIdx.z ? SV : SU;
    float out;
    if (rows == srows && cols == scols) {
        out = S.at(y, x);
    } else if (ix > 0 && iy > 0) {
        float acc = 0.f, grp[4];
        int k = 0;
        for (int dy = 0; dy < iy; ++dy)
            for (int dx = 0; dx < ix; ++dx) {
                grp[k++] = S.at(y * iy + dy, x * ix + dx);
                if (k == 4) {
                    acc = acc + (((grp[0] + grp[1]) + grp[2]) + grp[3]);
                    k = 0;
                }
            }
        for (int i = 0; i < k; ++i) acc = acc + grp[i];
        out = acc * (1.f / static_cast<float>(ix * iy));
    } else {
        const AreaAxis ax = area_axis(x, sx, scols), ay = area_axis(y, sy, srows);
        float acc = 0.f;
        bool first = true;
        for (int r = (ay.lo >= 0 ? ay.lo : ay.s1); r <= (ay.hi >= 0 ? ay.hi : ay.s2 - 1); ++r) {
            const float b = r == ay.lo ? ay.wlo : (r == ay.hi && r >= ay.s2) ? ay.whi : ay.wmid;
            float buf = 0.f;
            if (ax.lo >= 0) buf = buf + S.at(r, ax.lo) * ax.wlo;
            for (int c = ax.s1; c < ax.s2; ++c) buf = buf + S.at(r, c) * ax.wmid;
            if (ax.hi >= 0) buf = buf + S.at(r, ax.hi) * ax.whi;
            acc = first ? b * buf : acc + b * buf;
            first = false;
        }
        out = acc;
    }
    (blockIdx.z ? V : U).at(y, x) = apply_mul ? scale_val(out, mul) : out;
}

// ---------------------------------------------------------------------------------------------------------------
// Host tables
// ---------------------------------------------------------------------------------------------------------------

// getGaussianKernel(n, sigma, CV_32F)
void gaussian_kernel(int n, double sigma, float *out) {
    static const double f3[] = {0.25, 0.5, 0.25}, f5[] = {0.0625, 0.25, 0.375, 0.25, 0.0625},
                        f7[] = {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125};
    if (sigma <= 0 && (n == 1 || n == 3 || n == 5 || n == 7)) {
        const double *f = n == 3 ? f3 : n == 5 ? f5 : f7;
        for (int i = 0; i < n; ++i) out[i] = n == 1 ? 1.f : static_cast<float>(f[i]);
        return;
    }
    const double sx = sigma > 0 ? sigma : n * 0.15 + 0.35;
    const double s2 = -0.125 / (sx * sx);
    const int h = (n - 1) / 2;
    std::vector<double> vals(h);
    double sum = 0;
    for (int i = 0, x = 1 - n; i < h; ++i, x += 2) {
        vals[i] = std::exp(static_cast<double>(x * x) * s2);
        sum += vals[i];
    }
    sum = sum * 2.0 + 1.0 + (n % 2 == 0 ? 1.0 : 0.0);
    const double mul = 1.0 / sum;
    for (int i = 0; i < h; ++i) out[i] = out[n - 1 - i] = static_cast<float>(vals[i] * mul);
    out[h] = static_cast<float>(mul);
    if (n % 2 == 0) out[h + 1] = out[h];
}

// FarnebackPrepareGaussian: float taps, double moment sums and their Cholesky inverse (cv::invert DECOMP_CHOLESKY)
void poly_taps(int n, double sigma, PolyTaps &t) {
    if (sigma < FLT_EPSILON) sigma = n * 0.3;
    float *g = t.g + n, *xg = t.xg + n, *xxg = t.xxg + n;
    double s = 0.;
    for (int x = -n; x <= n; ++x) {
        g[x] = static_cast<float>(std::exp(-x * x / (2 * sigma * sigma)));
        s += g[x];
    }
    s = 1. / s;
    for (int x = -n; x <= n; ++x) {
        g[x] = static_cast<float>(g[x] * s);
        xg[x] = static_cast<float>(x * g[x]);
        xxg[x] = static_cast<float>(x * x * g[x]);
    }
    double G[6][6] = {};
    for (int y = -n; y <= n; ++y)
        for (int x = -n; x <= n; ++x) {
            const float fx = static_cast<float>(x), fy = static_cast<float>(y);
            const float gyx = g[y] * g[x];
            G[0][0] += gyx;
            G[1][1] += (gyx * fx) * fx;
            G[3][3] += (((gyx * fx) * fx) * fx) * fx;
            G[5][5] += (((gyx * fx) * fx) * fy) * fy;
        }
    G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
    G[4][4] = G[3][3];
    G[3][4] = G[4][3] = G[5][5];
    double L[6][6], B[6][6];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            L[i][j] = G[i][j];
            B[i][j] = i == j ? 1.0 : 0.0;
        }
    for (int i = 0; i < 6; ++i) {
        for (int j = 0; j < i; ++j) {
            double v = L[i][j];
            for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
            L[i][j] = v * L[j][j];
        }
        double v = L[i][i];
        for (int k = 0; k < i; ++k) v -= L[i][k] * L[i][k];
        L[i][i] = 1. / std::sqrt(v);
    }
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
            double v = B[i][j];
            for (int k = 0; k < i; ++k) v -= L[i][k] * B[k][j];
            B[i][j] = v * L[i][i];
        }
    for (int i = 5; i >= 0; --i)
        for (int j = 0; j < 6; ++j) {
            double v = B[i][j];
            for (int k = 5; k > i; --k) v -= L[k][i] * B[k][j];
            B[i][j] = v * L[i][i];
        }
    t.ig11 = B[1][1];
    t.ig03 = B[0][3];
    t.ig33 = B[3][3];
    t.ig55 = B[5][5];
    t.n = n;
}

// FarnebackUpdateFlow_GaussianBlur's window taps 0..m
void win_taps(int m, WinTaps &t) {
    const double sigma = m * 0.3;
    double s = 1;
    t.k[0] = 1.f;
    for (int i = 1; i <= m; ++i) {
        const float v = static_cast<float>(std::exp(-i * i / (2 * sigma * sigma)));
        t.k[i] = v;
        s += v * 2;
    }
    s = 1. / s;
    for (int i = 0; i <= m; ++i) t.k[i] = static_cast<float>(t.k[i] * s);
    t.m = m;
}

// resize.cpp's integer-factor test: 1 / (dst / src) within DBL_EPSILON of an integer
int exact_factor(int src, int dst) {
    const double s = 1.0 / (static_cast<double>(dst) / src);
    const int i = static_cast<int>(s);
    return std::fabs(s - i) < DBL_EPSILON ? i : 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Engine
// ---------------------------------------------------------------------------------------------------------------
class OptflowGFEngine : public b2f_handle {
public:
    explicit OptflowGFEngine(const b2f_farneback_params &p) : P(p) { algo = ALGO_OPTFLOWGF; }
    ~OptflowGFEngine() override {
        if (done_) cudaEventDestroy(done_);
    }
    b2f_farneback_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    const char *default_name() const override { return "DenseOpticalFlow.FarnebackOpticalFlow"; }
    bool reads_flow() const override { return (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) != 0; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"optflowgf_level", "optflowgf_poly", "optflowgf_update", "optflowgf_solve",
                                  "optflowgf_io"};
        return (cls >= 0 && cls < 5) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        Layout L;
        return layout(rows, cols, gauss(), initial(), true, L);
    }

private:
    // full-size: converted frames F, row-blurred T, the caller's flow UI / VI (OPTFLOW_USE_INITIAL_FLOW only);
    // level-size (allocated at level 0's): level images I, vertical poly sums RV (3 per frame), R0 / R1, M, the gaussian
    // window's float sums G (gaussian only), flow U / V and the previous level's PU / PV; and the box window's double
    // vertical sums vs (box only)
    enum { S_F0 = 0, S_F1, S_T0, S_T1, S_UI, S_VI, S_I0, S_I1, S_RV, S_R0 = S_RV + 6, S_R1 = S_R0 + 5, S_M = S_R1 + 5,
           S_G = S_M + 5, S_U = S_G + 5, S_V, S_PU, S_PV, S_COUNT };
    struct Layout {
        int rows = 0, cols = 0;
        bool gauss = false, initial = false;
        float *planes[S_COUNT] = {};
        double *vs = nullptr;
        size_t rpitch = 0;  // doubles between two columns of vs
    };
    Layout L_;
    struct GraphKey {
        int rows, cols;
        b2f_farneback_params P;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;

    // a handle may be called on several streams: a call on another stream than the previous one first waits for the
    // previous call, since both use this handle's workspace
    cudaEvent_t done_ = nullptr;
    cudaStream_t last_stream_ = nullptr;

    bool gauss() const { return (P.flags & B2F_OPTFLOW_FARNEBACK_GAUSSIAN) != 0; }
    bool initial() const { return (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) != 0; }
    size_t layout(int rows, int cols, bool gauss, bool initial, bool counting, Layout &L);
    cudaError_t ensure_workspace(int rows, int cols);
    Plane sp(int idx) const { return Plane{L_.planes[idx], plane_pitch(L_.cols)}; }
    Planes5 p5(int idx) const {
        Planes5 r;
        for (int i = 0; i < 5; ++i) r.p[i] = sp(idx + i);
        return r;
    }
    void solve(Ctx &c);
};

size_t OptflowGFEngine::layout(int rows, int cols, bool gauss, bool initial, bool counting, Layout &L) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.rows = rows;
    L.cols = cols;
    L.gauss = gauss;
    L.initial = initial;
    for (int i = 0; i < S_COUNT; ++i) {
        const bool unused = (!gauss && i >= S_G && i < S_G + 5) || (!initial && (i == S_UI || i == S_VI));
        L.planes[i] = unused ? nullptr : A.plane(rows, cols).p;
    }
    L.rpitch = (size_t)round_up(rows, 32);
    L.vs = gauss ? nullptr : static_cast<double *>(A.bytes(sizeof(double) * 5 * (size_t)cols * L.rpitch));
    return A.used();
}

cudaError_t OptflowGFEngine::ensure_workspace(int rows, int cols) {
    if (L_.rows == rows && L_.cols == cols && L_.gauss == gauss() && L_.initial == initial() && arena.capacity() > 0)
        return cudaSuccess;
    Layout tmp;
    const size_t need = layout(rows, cols, gauss(), initial(), true, tmp);
    graph_.destroy();
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    layout(rows, cols, gauss(), initial(), false, L_);
    return cudaSuccess;
}

void OptflowGFEngine::solve(Ctx &c) {
    const int rows = L_.rows, cols = L_.cols, pitch = plane_pitch(cols);
    const bool gauss = (P.flags & B2F_OPTFLOW_FARNEBACK_GAUSSIAN) != 0;
    int levels = 0;
    double scale = 1;
    for (; levels < P.num_levels; ++levels) {
        scale *= P.pyr_scale;
        if (cols * scale < 32 || rows * scale < 32) break;
    }
    PolyTaps pt;
    poly_taps(P.poly_n, P.poly_sigma, pt);
    WinTaps wt;
    const int m = P.win_size / 2;
    win_taps(gauss ? m : 0, wt);
    active_paths.assign(levels + 1, 0.0);
    int prows = 0, pcols = 0;
    const double bytes_px = 4.0;
    for (int k = levels; k >= 0; --k) {
        scale = 1;
        for (int i = 0; i < k; ++i) scale *= P.pyr_scale;
        const double sigma = (1. / scale - 1) * 0.5;
        const int ks = std::max(cv_round(sigma * 5) | 1, 3);
        const int w = cv_round(cols * scale), h = cv_round(rows * scale);
        BlurTaps bt;
        bt.ksize = ks;
        gaussian_kernel(ks, sigma, bt.k);
        const int level_mode = (w == cols && h == rows) ? 0
                               : (exact_factor(cols, w) == 2 && exact_factor(rows, h) == 2) ? 2 : 1;
        // the row blur only at the two columns each level column reads, when that is fewer than the frame's
        const int compact = level_mode == 1 && 2 * w < cols ? 1 : 0, tcols = compact ? 2 * w : cols;
        const double sx = 1.0 / (static_cast<double>(w) / cols), sy = 1.0 / (static_cast<double>(h) / rows);
        const dim3 blk(BS), full((tcols + BS - 1) / BS, rows, 2), lvl((w + BS - 1) / BS, h, 2);
        const dim3 lvl1((w + BS - 1) / BS, h, 1);
        B2F_LAUNCH(c, CLS_LEVEL, bytes_px * 2 * rows * (tcols + cols), k_gf_blur_rows, full, blk, 0, sp(S_F0), sp(S_F1),
                   sp(S_T0), sp(S_T1), cols, tcols, compact, sx, bt);
        B2F_LAUNCH(c, CLS_LEVEL, bytes_px * 2 * w * h * (2 * ks + 1), k_gf_level, lvl, blk, 0, sp(S_T0), sp(S_T1),
                   sp(S_I0), sp(S_I1), rows, cols, w, level_mode, compact, sx, sy, bt);
        // level-size planes use the full-size pitch
        Planes3x2 rv;
        for (int i = 0; i < 6; ++i) rv.p[i] = sp(S_RV + i);
        B2F_LAUNCH(c, CLS_POLY, bytes_px * 8 * w * h, k_gf_poly_v, lvl, blk, 0, sp(S_I0), sp(S_I1), rv, h, w, pt);
        B2F_LAUNCH(c, CLS_POLY, bytes_px * 16 * w * h, k_gf_poly_h, lvl, blk, 0, rv, p5(S_R0), p5(S_R1), w, pt);
        if (prows == 0) {
            if (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) {
                B2F_LAUNCH(c, CLS_IO, bytes_px * 2 * (rows * cols + w * h), k_gf_area, lvl, blk, 0, sp(S_UI), sp(S_VI),
                           sp(S_U), sp(S_V), rows, cols, h, w, exact_factor(cols, w), exact_factor(rows, h),
                           1.0 / (static_cast<double>(w) / cols), 1.0 / (static_cast<double>(h) / rows),
                           static_cast<float>(scale), scale != 1.0 ? 1 : 0);
            } else {
                if (c.ok()) c.check(cudaMemsetAsync(L_.planes[S_U], 0, sizeof(float) * (size_t)pitch * h, c.stream));
                if (c.ok()) c.check(cudaMemsetAsync(L_.planes[S_V], 0, sizeof(float) * (size_t)pitch * h, c.stream));
            }
        } else {
            const int pmode = (w == pcols && h == prows) ? 0 : 1;
            B2F_LAUNCH(c, CLS_IO, bytes_px * 4 * w * h, k_gf_prolong, lvl, blk, 0, sp(S_PU), sp(S_PV), sp(S_U), sp(S_V),
                       prows, pcols, h, w, pmode, 1.0 / (static_cast<double>(w) / pcols),
                       1.0 / (static_cast<double>(h) / prows), static_cast<float>(1. / P.pyr_scale));
        }
        const dim3 lvl5((w + BS - 1) / BS, h, 5);
        B2F_LAUNCH(c, CLS_UPDATE, bytes_px * 32 * w * h, k_gf_update, lvl1, blk, 0, p5(S_R0), p5(S_R1), sp(S_U), sp(S_V),
                   p5(S_M), h, w);
        for (int it = 0; it < P.num_iters; ++it) {
            if (gauss) {
                B2F_LAUNCH(c, CLS_SOLVE, bytes_px * 10 * w * h * (m + 1), k_gf_gauss_v, lvl5, blk, 0, p5(S_M), p5(S_G), h,
                           w, wt);
                B2F_LAUNCH(c, CLS_SOLVE, bytes_px * 10 * w * h * (m + 1), k_gf_gauss_h, lvl1, blk, 0, p5(S_G), sp(S_U),
                           sp(S_V), w, wt);
            } else {
                const size_t cstride = (size_t)cols * L_.rpitch;
                B2F_LAUNCH(c, CLS_SOLVE, bytes_px * 15 * w * h, k_gf_box_v, dim3((w + BOX_TILE - 1) / BOX_TILE, 5),
                           dim3(BOX_TILE), 0, p5(S_M), L_.vs, cstride, L_.rpitch, h, w, m);
                B2F_LAUNCH(c, CLS_SOLVE, bytes_px * 22 * w * h, k_gf_box_h, dim3((h + 31) / 32), dim3(32), 0, L_.vs,
                           cstride, L_.rpitch, sp(S_U), sp(S_V), h, w, m, 1. / (P.win_size * P.win_size));
            }
            if (it < P.num_iters - 1)
                B2F_LAUNCH(c, CLS_UPDATE, bytes_px * 32 * w * h, k_gf_update, lvl1, blk, 0, p5(S_R0), p5(S_R1), sp(S_U),
                           sp(S_V), p5(S_M), h, w);
        }
        // B2F_ENGINE_ACTIVE_PATH per level, finest first: the window (B2F_OPTFLOWGF_PATH_BOX / _GAUSSIAN), plus
        // B2F_OPTFLOWGF_PATH_AREA_LEVEL when the level images took the exact-half fast-area rule
        active_paths[k] = (gauss ? B2F_OPTFLOWGF_PATH_GAUSSIAN : B2F_OPTFLOWGF_PATH_BOX) |
                          (level_mode == 2 ? B2F_OPTFLOWGF_PATH_AREA_LEVEL : 0);
        if (k > 0) {
            if (c.ok()) c.check(cudaMemcpyAsync(L_.planes[S_PU], L_.planes[S_U], sizeof(float) * (size_t)pitch * h,
                                                cudaMemcpyDeviceToDevice, c.stream));
            if (c.ok()) c.check(cudaMemcpyAsync(L_.planes[S_PV], L_.planes[S_V], sizeof(float) * (size_t)pitch * h,
                                                cudaMemcpyDeviceToDevice, c.stream));
        }
        prows = h;
        pcols = w;
    }
    if (c.stats) c.stats->iterations_run = P.num_iters * (levels + 1);
}

int OptflowGFEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    if ((I0->type != B2F_8UC1 && I0->type != B2F_32FC1) || I1->type != I0->type) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (I0->rows <= 0 || I0->cols <= 0) return B2F_BAD_ARG;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    // cv2 asserts pyrScale < 1; the kernels hold polyN 1..B2F_OPTFLOWGF_MAX_POLY_N and winSize 1..B2F_OPTFLOWGF_MAX_WIN_SIZE
    if (!(P.pyr_scale < 1) || P.poly_n < 1 || P.poly_n > GF_MAX_POLY_N || P.win_size < 1 || P.win_size > GF_MAX_WIN)
        return B2F_BAD_ARG;
    const size_t esz = I0->type == B2F_8UC1 ? 1 : 4;
    if (I0->step < (size_t)I0->cols * esz || I1->step < (size_t)I1->cols * esz || !flow_step_ok(flow)) return B2F_BAD_ARG;
    const int rows = I0->rows, cols = I0->cols;
    {  // the deepest level's blur must fit the tap table
        int levels = 0;
        double scale = 1;
        for (; levels < P.num_levels; ++levels) {
            scale *= P.pyr_scale;
            if (cols * scale < 32 || rows * scale < 32) break;
        }
        scale = 1;
        for (int i = 0; i < levels; ++i) scale *= P.pyr_scale;
        if (std::max(cv_round((1. / scale - 1) * 0.5 * 5) | 1, 3) > GF_MAX_BLUR) return B2F_BAD_ARG;
    }
    Ctx c = make_ctx(s);
    cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
    if (s && cudaStreamIsCapturing(s, &capturing) != cudaSuccess) cudaGetLastError();
    const bool caller_capture = capturing != cudaStreamCaptureStatusNone;
    // order after the previous call when it ran on another stream (inside a caller's capture the caller orders)
    if (!caller_capture && done_ && last_stream_ != s) c.check(cudaStreamWaitEvent(s, done_, 0));
    c.check(ensure_workspace(rows, cols));
    if (!c.ok()) return finish(c, s);
    stats.iterations_run = 0;

    // the caller's images and flow are read before the graph, which must not bake their addresses in
    const ImageView a{I0->data, I0->step, rows, cols, I0->type}, b{I1->data, I1->step, rows, cols, I1->type};
    convert_pair(c, CLS_IO, a, b, sp(S_F0), sp(S_F1), 1.0f);
    const ImageView vf = flow_view(flow, rows, cols);
    if (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) split_flow(c, CLS_IO, vf, sp(S_UI), sp(S_VI));
    const bool want_graph = knobs.use_graph && !profiling && s != nullptr;
    if (want_graph) {
        graph_.run(*this, c, s, GraphKey{rows, cols, P, L_.planes[0]}, [&](Ctx &g) { solve(g); });
    } else {
        solve(c);
    }
    stats.levels = static_cast<int>(active_paths.size());
    merge_flow(c, CLS_IO, sp(S_U), sp(S_V), vf);
    if (!caller_capture && c.ok()) {
        if (!done_) c.check(cudaEventCreateWithFlags(&done_, cudaEventDisableTiming));
        if (c.ok()) c.check(cudaEventRecord(done_, s));
        last_stream_ = s;
    }
    return finish(c, s);
}

int OptflowGFEngine::set_param(int id, double v) {
    switch (id) {
        case B2F_FARN_NUM_LEVELS: P.num_levels = static_cast<int>(v); break;
        case B2F_FARN_PYR_SCALE: P.pyr_scale = v; break;
        case B2F_FARN_FAST_PYRAMIDS: P.fast_pyramids = v != 0; break;
        case B2F_FARN_WIN_SIZE: P.win_size = static_cast<int>(v); break;
        case B2F_FARN_NUM_ITERS: P.num_iters = static_cast<int>(v); break;
        case B2F_FARN_POLY_N: P.poly_n = static_cast<int>(v); break;
        case B2F_FARN_POLY_SIGMA: P.poly_sigma = v; break;
        case B2F_FARN_FLAGS: P.flags = static_cast<int>(v); break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

int OptflowGFEngine::get_param(int id, double *v) const {
    switch (id) {
        case B2F_FARN_NUM_LEVELS: *v = P.num_levels; break;
        case B2F_FARN_PYR_SCALE: *v = P.pyr_scale; break;
        case B2F_FARN_FAST_PYRAMIDS: *v = P.fast_pyramids; break;
        case B2F_FARN_WIN_SIZE: *v = P.win_size; break;
        case B2F_FARN_NUM_ITERS: *v = P.num_iters; break;
        case B2F_FARN_POLY_N: *v = P.poly_n; break;
        case B2F_FARN_POLY_SIGMA: *v = P.poly_sigma; break;
        case B2F_FARN_FLAGS: *v = P.flags; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

}  // namespace
}  // namespace b2f

extern "C" {

int b2f_optflowgf_create(const b2f_farneback_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_farneback_params d;
    b2f_farneback_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::OptflowGFEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
