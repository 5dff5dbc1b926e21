// lkpyramid.cu -- the video module's pyramidal Lucas-Kanade tracker: cv::buildOpticalFlowPyramid and
// cv::calcOpticalFlowPyrLK / cv::SparsePyrLKOpticalFlow, bit for bit equal to cv2 4.13's x86 build (oracle/lkpyramid_model.py
// states every rounding and the summation order; DESIGN §4.13).
//
// Pyramid: uint8 levels of cn interleaved channels, each stored with a (win_w, win_h) BORDER_REFLECT_101 border, level
// sizes ((w + 1) / 2, (h + 1) / 2) by cv::pyrDown's integer 5x5 filter; optional int16 Scharr derivatives (Ix, Iy per
// channel) with a zero (BORDER_CONSTANT) border.  Tracker: one thread per point walks every level inside one launch with
// cv2's fixed-point bilinear taps (W_BITS 14), and adds its float sums in cv2's SIMD lane order.  Built with -fmad=false,
// so every float expression rounds once per operation as the model does.
#include <algorithm>
#include <climits>
#include <cstring>
#include <new>

#include "common.cuh"

namespace b2f {
namespace {

constexpr int LK_MAX_LEVELS = 16;
constexpr int LK_BLOCK = 32;  // one warp per block, so that a few thousand points spread over many SMs
enum { CLS_PYR = 0, CLS_DERIV = 1, CLS_TRACK = 2 };

__device__ __forceinline__ int reflect101(int p, int n) {
    if (n == 1) return 0;
    while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * (n - 1) - p;
    return p;
}

// padded level 0 from the caller's image: every padded pixel takes the reflect-101 image pixel
__global__ void __launch_bounds__(256) k_lk_pad(const unsigned char *__restrict__ src, size_t sstep, int rows, int cols,
                                                 int cn, unsigned char *__restrict__ dst, size_t dstep, int bw, int bh) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols + 2 * bw || y >= rows + 2 * bh) return;
    const unsigned char *s = src + (size_t)reflect101(y - bh, rows) * sstep + (size_t)reflect101(x - bw, cols) * cn;
    unsigned char *d = dst + (size_t)y * dstep + (size_t)x * cn;
    for (int c = 0; c < cn; ++c) d[c] = s[c];
}

// cv::pyrDown for 8U into a padded level: (sum of [1 4 6 4 1]^2 taps + 128) >> 8, reflect-101 of the source; the border
// pixels are the reflect-101 interior pixels
__global__ void __launch_bounds__(256) k_lk_pyrdown(const unsigned char *__restrict__ src, size_t sstep, int srows, int scols,
                                                     int cn, unsigned char *__restrict__ dst, size_t dstep, int rows, int cols,
                                                     int bw, int bh) {
    const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (px >= cols + 2 * bw || py >= rows + 2 * bh) return;
    const int x = reflect101(px - bw, cols), y = reflect101(py - bh, rows);
    const int k[5] = {1, 4, 6, 4, 1};
    int sx[5], sy[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        sx[i] = reflect101(2 * x + i - 2, scols);
        sy[i] = reflect101(2 * y + i - 2, srows);
    }
    for (int c = 0; c < cn; ++c) {
        int v = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const unsigned char *r = src + (size_t)sy[i] * sstep + c;
            int h = 0;
#pragma unroll
            for (int j = 0; j < 5; ++j) h += k[j] * r[(size_t)sx[j] * cn];
            v += k[i] * h;
        }
        dst[(size_t)py * dstep + (size_t)px * cn + c] = (unsigned char)((v + 128) >> 8);
    }
}

// calcSharrDeriv into a padded int16 (Ix, Iy) x cn plane with a zero border
__global__ void __launch_bounds__(256) k_lk_scharr(const unsigned char *__restrict__ src, size_t sstep, int rows, int cols, int cn,
                                                    short *__restrict__ dst, size_t dstep, int bw, int bh) {
    const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (px >= cols + 2 * bw || py >= rows + 2 * bh) return;
    short *d = reinterpret_cast<short *>(reinterpret_cast<char *>(dst) + (size_t)py * dstep) + (size_t)px * 2 * cn;
    const int x = px - bw, y = py - bh;
    if (x < 0 || x >= cols || y < 0 || y >= rows) {
        for (int c = 0; c < 2 * cn; ++c) d[c] = 0;
        return;
    }
    const int ym = reflect101(y - 1, rows), yp = reflect101(y + 1, rows);
    const int xm = reflect101(x - 1, cols), xp = reflect101(x + 1, cols);
    const unsigned char *r0 = src + (size_t)ym * sstep, *r1 = src + (size_t)y * sstep, *r2 = src + (size_t)yp * sstep;
    for (int c = 0; c < cn; ++c) {
        auto t0 = [&](int xx) { return (int)(short)((r0[xx * cn + c] + r2[xx * cn + c]) * 3 + r1[xx * cn + c] * 10); };
        auto t1 = [&](int xx) { return (int)(short)(r2[xx * cn + c] - r0[xx * cn + c]); };
        d[2 * c] = (short)(t0(xp) - t0(xm));
        d[2 * c + 1] = (short)((t1(xp) + t1(xm)) * 3 + t1(x) * 10);
    }
}

struct LkLevel {
    const unsigned char *I;  // interior (0, 0) of the padded prev level
    const short *dI;         // interior (0, 0) of the padded derivative level
    const unsigned char *J;  // interior (0, 0) of the padded next level
    int istep, dstep, jstep;  // elements (bytes for I / J, shorts for dI)
    int rows, cols;
};
struct LkLevels {
    LkLevel l[LK_MAX_LEVELS];
};
struct LkArgs {
    int win_w, win_h, cn, max_level, max_count, flags;
    double eps;  // squared, as calcOpticalFlowPyrLK stores it
    float min_eig;
};

// cvFloor; NaN and values outside int32 give x86's integer-indefinite INT_MIN, which every window test rejects
__device__ __forceinline__ int lk_floor(float v) {
    if (!(v >= -2147483648.f && v < 2147483648.f)) return INT_MIN;
    return (int)floorf(v);
}
__device__ __forceinline__ bool lk_outside(int ix, int iy, const LkArgs &A, const LkLevel &L) {
    return ix < -A.win_w || ix >= L.cols || iy < -A.win_h || iy >= L.rows;
}
__device__ __forceinline__ void lk_weights(float a, float b, int &w00, int &w01, int &w10, int &w11) {
    w00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
    w01 = __float2int_rn(a * (1.f - b) * 16384.f);
    w10 = __float2int_rn((1.f - a) * b * 16384.f);
    w11 = (1 << 14) - w00 - w01 - w10;
}
// element x of the bilinear 8-bit patch, scaled by 32: CV_DESCALE(..., W_BITS - 5)
__device__ __forceinline__ int lk_pix(const unsigned char *r, int step, int x, int cn, int w00, int w01, int w10, int w11) {
    return ((int)r[x] * w00 + (int)r[x + cn] * w01 + (int)r[x + step] * w10 + (int)r[x + step + cn] * w11 + (1 << 8)) >> 9;
}
__device__ __forceinline__ int lk_der(const short *r, int step, int k, int cn2, int w00, int w01, int w10, int w11) {
    return ((int)r[k] * w00 + (int)r[k + cn2] * w01 + (int)r[k + step] * w10 + (int)r[k + step + cn2] * w11 + (1 << 13)) >> 14;
}

// LKTrackerInvoker for every level of one point
__global__ void __launch_bounds__(LK_BLOCK) k_lk_track(LkLevels Ls, LkArgs A, const float2 *__restrict__ prev_pts,
                                                        float2 *__restrict__ next_pts, unsigned char *__restrict__ status,
                                                        float *__restrict__ err, int n) {
    const int pt = blockIdx.x * blockDim.x + threadIdx.x;
    if (pt >= n) return;
    const int ww = A.win_w, wh = A.win_h, cn = A.cn, cn2 = 2 * cn, nel = ww * cn;
    const int nA = nel >= 8 ? (nel / 8) * 8 : 0;  // the 8-wide SIMD part of each row, covariance
    const int nB = nA;                            // and mismatch loops
    const float hx = (float)(ww - 1) * 0.5f, hy = (float)(wh - 1) * 0.5f;
    const bool get_mineig = (A.flags & 8) != 0;
    const float2 p0 = prev_pts[pt];
    float2 out = next_pts[pt];
    unsigned char st = 1;
    float ev = 0.f;
    bool ev_set = false;

    for (int level = A.max_level; level >= 0; --level) {
        const LkLevel &L = Ls.l[level];
        const float sc = 1.f / (float)(1 << level);
        float2 prevPt = make_float2(p0.x * sc, p0.y * sc);
        float2 nextPt;
        if (level == A.max_level)
            nextPt = (A.flags & 4) ? make_float2(out.x * sc, out.y * sc) : prevPt;
        else
            nextPt = make_float2(out.x * 2.f, out.y * 2.f);
        out = nextPt;
        prevPt.x = prevPt.x - hx;
        prevPt.y = prevPt.y - hy;
        const int ipx = lk_floor(prevPt.x), ipy = lk_floor(prevPt.y);
        if (lk_outside(ipx, ipy, A, L)) {
            if (level == 0) {
                st = 0;
                ev = 0.f;
                ev_set = true;
            }
            continue;
        }
        int w00, w01, w10, w11;
        lk_weights(prevPt.x - (float)ipx, prevPt.y - (float)ipy, w00, w01, w10, w11);
        const unsigned char *Ib = L.I + (ptrdiff_t)ipy * L.istep + (ptrdiff_t)ipx * cn;
        const short *dIb = L.dI + (ptrdiff_t)ipy * L.dstep + (ptrdiff_t)ipx * cn2;

        float q11[4] = {0.f, 0.f, 0.f, 0.f}, q12[4] = {0.f, 0.f, 0.f, 0.f}, q22[4] = {0.f, 0.f, 0.f, 0.f};
        float s11 = 0.f, s12 = 0.f, s22 = 0.f;
        for (int y = 0; y < wh; ++y) {
            const short *dr = dIb + (ptrdiff_t)y * L.dstep;
            int x = 0;
            for (; x < nA; x += 8) {
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float fx = (float)lk_der(dr, L.dstep, 2 * (x + k), cn2, w00, w01, w10, w11);
                    const float fy = (float)lk_der(dr, L.dstep, 2 * (x + k) + 1, cn2, w00, w01, w10, w11);
                    q22[k & 3] = q22[k & 3] + fy * fy;
                    q12[k & 3] = q12[k & 3] + fx * fy;
                    q11[k & 3] = q11[k & 3] + fx * fx;
                }
            }
            for (; x < nel; ++x) {
                const int ix = lk_der(dr, L.dstep, 2 * x, cn2, w00, w01, w10, w11);
                const int iy = lk_der(dr, L.dstep, 2 * x + 1, cn2, w00, w01, w10, w11);
                s11 = s11 + (float)(ix * ix);
                s12 = s12 + (float)(ix * iy);
                s22 = s22 + (float)(iy * iy);
            }
        }
        const float FLT_SCALE = 1.f / (float)(1 << 20);
        const float A11 = (s11 + ((q11[0] + q11[2]) + (q11[1] + q11[3]))) * FLT_SCALE;
        const float A12 = (s12 + ((q12[0] + q12[2]) + (q12[1] + q12[3]))) * FLT_SCALE;
        const float A22 = (s22 + ((q22[0] + q22[2]) + (q22[1] + q22[3]))) * FLT_SCALE;
        float D = A11 * A22 - A12 * A12;
        const float minEig = ((A22 + A11) - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * ww * wh);
        if (get_mineig) {
            ev = minEig;
            ev_set = true;
        }
        if (minEig < A.min_eig || D < FLT_EPSILON) {
            if (level == 0) st = 0;
            continue;
        }
        D = 1.f / D;
        nextPt.x = nextPt.x - hx;
        nextPt.y = nextPt.y - hy;
        float2 prevDelta = make_float2(0.f, 0.f);
        for (int j = 0; j < A.max_count; ++j) {
            const int inx = lk_floor(nextPt.x), iny = lk_floor(nextPt.y);
            if (lk_outside(inx, iny, A, L)) {
                if (level == 0) st = 0;
                break;
            }
            int v00, v01, v10, v11;
            lk_weights(nextPt.x - (float)inx, nextPt.y - (float)iny, v00, v01, v10, v11);
            const unsigned char *Jb = L.J + (ptrdiff_t)iny * L.jstep + (ptrdiff_t)inx * cn;
            float q0[4] = {0.f, 0.f, 0.f, 0.f}, q1[4] = {0.f, 0.f, 0.f, 0.f};
            float ib1 = 0.f, ib2 = 0.f;
            for (int y = 0; y < wh; ++y) {
                const unsigned char *ir = Ib + (ptrdiff_t)y * L.istep, *jr = Jb + (ptrdiff_t)y * L.jstep;
                const short *dr = dIb + (ptrdiff_t)y * L.dstep;
                int x = 0;
                for (; x < nB; x += 8) {
                    int dif[8], gx[8], gy[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        dif[k] = lk_pix(jr, L.jstep, x + k, cn, v00, v01, v10, v11) - lk_pix(ir, L.istep, x + k, cn, w00, w01, w10, w11);
                        gx[k] = lk_der(dr, L.dstep, 2 * (x + k), cn2, w00, w01, w10, w11);
                        gy[k] = lk_der(dr, L.dstep, 2 * (x + k) + 1, cn2, w00, w01, w10, w11);
                    }
                    q0[0] = q0[0] + (float)(dif[0] * gx[0] + dif[4] * gx[4]);
                    q0[1] = q0[1] + (float)(dif[0] * gy[0] + dif[4] * gy[4]);
                    q0[2] = q0[2] + (float)(dif[1] * gx[1] + dif[5] * gx[5]);
                    q0[3] = q0[3] + (float)(dif[1] * gy[1] + dif[5] * gy[5]);
                    q1[0] = q1[0] + (float)(dif[2] * gx[2] + dif[6] * gx[6]);
                    q1[1] = q1[1] + (float)(dif[2] * gy[2] + dif[6] * gy[6]);
                    q1[2] = q1[2] + (float)(dif[3] * gx[3] + dif[7] * gx[7]);
                    q1[3] = q1[3] + (float)(dif[3] * gy[3] + dif[7] * gy[7]);
                }
                for (; x < nel; ++x) {
                    const int d = lk_pix(jr, L.jstep, x, cn, v00, v01, v10, v11) - lk_pix(ir, L.istep, x, cn, w00, w01, w10, w11);
                    ib1 = ib1 + (float)(d * lk_der(dr, L.dstep, 2 * x, cn2, w00, w01, w10, w11));
                    ib2 = ib2 + (float)(d * lk_der(dr, L.dstep, 2 * x + 1, cn2, w00, w01, w10, w11));
                }
            }
            const float b1 = (ib1 + ((q0[0] + q1[0]) + (q0[2] + q1[2]))) * FLT_SCALE;
            const float b2 = (ib2 + ((q0[1] + q1[1]) + (q0[3] + q1[3]))) * FLT_SCALE;
            const float dx = (A12 * b2 - A22 * b1) * D;
            const float dy = (A12 * b1 - A11 * b2) * D;
            nextPt.x = nextPt.x + dx;
            nextPt.y = nextPt.y + dy;
            out = make_float2(nextPt.x + hx, nextPt.y + hy);
            if ((double)dx * (double)dx + (double)dy * (double)dy <= A.eps) break;
            if (j > 0 && fabs((double)(dx + prevDelta.x)) < 0.01 && fabs((double)(dy + prevDelta.y)) < 0.01) {
                out.x = out.x - dx * 0.5f;
                out.y = out.y - dy * 0.5f;
                break;
            }
            prevDelta = make_float2(dx, dy);
        }

        if (st && level == 0 && !get_mineig && err) {
            const float nx = out.x - hx, ny = out.y - hy;
            const int inx = lk_floor(nx), iny = lk_floor(ny);
            if (lk_outside(inx, iny, A, L)) {
                st = 0;
                continue;
            }
            int v00, v01, v10, v11;
            lk_weights(nx - (float)inx, ny - (float)iny, v00, v01, v10, v11);
            const unsigned char *Jb = L.J + (ptrdiff_t)iny * L.jstep + (ptrdiff_t)inx * cn;
            float e = 0.f;
            for (int y = 0; y < wh; ++y) {
                const unsigned char *ir = Ib + (ptrdiff_t)y * L.istep, *jr = Jb + (ptrdiff_t)y * L.jstep;
                for (int x = 0; x < nel; ++x) {
                    const int d = lk_pix(jr, L.jstep, x, cn, v00, v01, v10, v11) - lk_pix(ir, L.istep, x, cn, w00, w01, w10, w11);
                    e = e + fabsf((float)d);
                }
            }
            ev = e / (float)(32 * ww * cn * wh);
            ev_set = true;
        }
    }
    next_pts[pt] = out;
    status[pt] = st;
    if (err && ev_set) err[pt] = ev;
}

// levels a buildOpticalFlowPyramid call keeps for an image of rows x cols (its return value)
int lk_levels(int rows, int cols, int ww, int wh, int max_level) {
    int w = cols, h = rows;
    for (int level = 0; level <= max_level; ++level) {
        w = (w + 1) / 2;
        h = (h + 1) / 2;
        if (w <= ww || h <= wh) return level;
    }
    return max_level;
}

// process-wide source of layout generations: no two layouts of any two pyramids share a value, so a graph key that
// holds a generation names that layout's device addresses even after the host object is freed and its address reused
std::atomic<uint64_t> g_lk_generation{0};

}  // namespace
}  // namespace b2f

// a device pyramid: padded uint8 levels and, optionally, padded int16 derivatives, in one arena
struct b2f_lkpyr_pyramid {
    b2f::Arena arena;
    int rows = 0, cols = 0, cn = 0, win_w = 0, win_h = 0, levels = 0, derivs = 0;
    uint64_t generation = 0;  // a fresh process-wide value on every layout (level addresses change)
    struct Lvl {
        unsigned char *img;  // padded origin
        short *der;          // padded origin or null
        size_t istep, dstep; // bytes
        int rows, cols;
    };
    std::vector<Lvl> L;

    // lays out (rows, cols, cn, win, levels, derivs); a grown arena waits for `s` first
    int layout(b2f::Ctx &c, int r, int cc, int ch, int bw, int bh, int nlev, int der) {
        using namespace b2f;
        if (r == rows && cc == cols && ch == cn && bw == win_w && bh == win_h && nlev == levels && der == derivs &&
            arena.capacity() > 0)
            return B2F_OK;
        for (int pass = 0; pass < 2 && c.ok(); ++pass) {
            Arena tmp;
            Arena &A = pass == 0 ? tmp : arena;
            A.begin(pass == 0);
            L.assign(nlev, Lvl{});
            int h = r, w = cc;
            for (int l = 0; l < nlev; ++l) {
                if (l) {
                    w = (w + 1) / 2;
                    h = (h + 1) / 2;
                }
                Lvl &v = L[l];
                v.rows = h;
                v.cols = w;
                v.istep = (size_t)round_up((w + 2 * bw) * ch, 128);
                v.img = static_cast<unsigned char *>(A.bytes(v.istep * (h + 2 * bh)));
                v.dstep = der ? (size_t)round_up((w + 2 * bw) * 2 * ch * 2, 128) : 0;
                v.der = der ? static_cast<short *>(A.bytes(v.dstep * (h + 2 * bh))) : nullptr;
            }
            if (pass == 0) {
                if (A.used() > arena.capacity() && arena.capacity() > 0) c.check(cudaStreamSynchronize(c.stream));
                c.check(arena.reserve(A.used()));
            }
        }
        if (!c.ok()) return B2F_CUDA_ERROR;
        rows = r; cols = cc; cn = ch; win_w = bw; win_h = bh; levels = nlev; derivs = der;
        generation = ++b2f::g_lk_generation;
        return B2F_OK;
    }

    void launch_deriv(b2f::Ctx &c, int l) {
        using namespace b2f;
        const Lvl &v = L[l];
        const dim3 blk(32, 8), grid(div_up(v.cols + 2 * win_w, 32), div_up(v.rows + 2 * win_h, 8));
        B2F_LAUNCH(c, CLS_DERIV, (double)(v.rows + 2 * win_h) * (v.cols + 2 * win_w) * cn * 5.0, k_lk_scharr, grid, blk, 0,
                   v.img + (size_t)win_h * v.istep + (size_t)win_w * cn, v.istep, v.rows, v.cols, cn, v.der, v.dstep, win_w, win_h);
    }

    // every level from a caller's image
    void build(b2f::Ctx &c, const b2f_image *img) {
        using namespace b2f;
        const dim3 blk(32, 8);
        for (int l = 0; l < levels; ++l) {
            const Lvl &v = L[l];
            const dim3 grid(div_up(v.cols + 2 * win_w, 32), div_up(v.rows + 2 * win_h, 8));
            const double bytes = (double)(v.rows + 2 * win_h) * (v.cols + 2 * win_w) * cn * 2.0;
            if (l == 0) {
                B2F_LAUNCH(c, CLS_PYR, bytes, k_lk_pad, grid, blk, 0, static_cast<const unsigned char *>(img->data), img->step,
                           rows, cols, cn, v.img, v.istep, win_w, win_h);
            } else {
                const Lvl &s = L[l - 1];
                B2F_LAUNCH(c, CLS_PYR, bytes, k_lk_pyrdown, grid, blk, 0, s.img + (size_t)win_h * s.istep + (size_t)win_w * cn,
                           s.istep, s.rows, s.cols, cn, v.img, v.istep, v.rows, v.cols, win_w, win_h);
            }
            if (derivs) launch_deriv(c, l);
        }
    }
};

struct b2f_lkpyr : b2f_handle {
    b2f_lkpyr_params P{};
    b2f_lkpyr_pyramid own_prev, own_next, own_deriv;  // images' pyramids; derivatives of a pyramid built without them
    // The workspace is shared by every call of the handle: a call on another stream than the previous one first waits
    // for the previous call's work (recorded in `done`), so that it cannot rewrite pyramids a tracker is still reading.
    cudaEvent_t done = nullptr;
    cudaStream_t last_stream = nullptr;
    ~b2f_lkpyr() override {
        if (done) cudaEventDestroy(done);
    }

    // The graph is used only when both frames are images: everything it bakes in is then the caller's image and point
    // pointers plus the handle's own arenas, whose layout generations are process-wide unique.  A caller's pyramids
    // (their addresses rotate in a frame loop) go through direct launches and are never baked into a graph.
    struct Key {
        const void *prev = nullptr, *next = nullptr, *pp = nullptr, *np = nullptr, *st = nullptr, *err = nullptr;
        uint64_t gen[2] = {};
        size_t pstep = 0, nstep = 0;
        int rows = 0, cols = 0, type = 0, n = 0, max_level = 0, win_w = 0, win_h = 0, max_count = 0, flags = 0;
        double eps = 0, min_eig = 0;
        bool operator==(const Key &o) const {
            return gen[0] == o.gen[0] && gen[1] == o.gen[1] && prev == o.prev && next == o.next && pp == o.pp && np == o.np &&
                   st == o.st && err == o.err && pstep == o.pstep && nstep == o.nstep &&
                   rows == o.rows && cols == o.cols && type == o.type && n == o.n && max_level == o.max_level &&
                   win_w == o.win_w && win_h == o.win_h && max_count == o.max_count && flags == o.flags && eps == o.eps &&
                   min_eig == o.min_eig;
        }
    };
    b2f::GraphCache<Key> graph;

    int calc(const b2f_image *, const b2f_image *, b2f_image *, cudaStream_t) override { return B2F_BAD_ARG; }
    int set_param(int, double) override { return B2F_BAD_ARG; }
    int get_param(int, double *) const override { return B2F_BAD_ARG; }
    const char *default_name() const override { return "SparsePyrLKOpticalFlow"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"lk_pyramid", "lk_scharr", "lk_track"};
        return cls >= 0 && cls < 3 ? n[cls] : "";
    }
    size_t workspace_bytes(int, int, int) override {
        return own_prev.arena.capacity() + own_next.arena.capacity() + own_deriv.arena.capacity();
    }
};

namespace {

int lk_image_ok(const b2f_image *im) {
    if (!im || !im->data || im->rows < 1 || im->cols < 1) return B2F_BAD_ARG;
    if (im->type < 0 || (im->type & 7) != 0) return B2F_UNSUPPORTED_TYPE;  // CV_Assert(depth == CV_8U)
    const int cn = (im->type >> 3) + 1;
    if (cn > 256) return B2F_UNSUPPORTED_TYPE;  // derivatives are CV_16SC(2 cn), at most CV_CN_MAX channels
    if (im->step < (size_t)im->cols * cn) return B2F_BAD_ARG;
    return B2F_OK;
}

bool lk_params_ok(const b2f_lkpyr_params &p) {
    return p.win_width > 2 && p.win_height > 2 && p.max_level >= 0;  // lkpyramid.cpp's CV_Asserts
}

}  // namespace

extern "C" {

void b2f_lkpyr_default_params(b2f_lkpyr_params *p) {
    if (!p) return;
    p->win_width = 21;
    p->win_height = 21;
    p->max_level = 3;
    p->criteria_type = 3;  // TermCriteria::COUNT + TermCriteria::EPS
    p->max_count = 30;
    p->epsilon = 0.01;
    p->flags = 0;
    p->min_eig_threshold = 1e-4;
}

int b2f_lkpyr_create(const b2f_lkpyr_params *p, b2f_lkpyr **out) {
    if (!out) return B2F_BAD_ARG;
    *out = nullptr;
    b2f_lkpyr_params P;
    b2f_lkpyr_default_params(&P);
    if (p) P = *p;
    if (!lk_params_ok(P)) return B2F_BAD_ARG;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return B2F_NO_DEVICE;
    }
    auto *h = new (std::nothrow) b2f_lkpyr();
    if (!h) return B2F_OUT_OF_MEMORY;
    h->P = P;
    *out = h;
    return B2F_OK;
}

int b2f_lkpyr_set_params(b2f_lkpyr *h, const b2f_lkpyr_params *p) {
    if (!h || !p || !lk_params_ok(*p)) return B2F_BAD_ARG;
    h->P = *p;
    return B2F_OK;
}

int b2f_lkpyr_get_params(const b2f_lkpyr *h, b2f_lkpyr_params *p) {
    if (!h || !p) return B2F_BAD_ARG;
    *p = h->P;
    return B2F_OK;
}

b2f_handle *b2f_lkpyr_engine(b2f_lkpyr *h) { return h; }

int b2f_lkpyr_pyramid_create(b2f_lkpyr_pyramid **out) {
    if (!out) return B2F_BAD_ARG;
    *out = new (std::nothrow) b2f_lkpyr_pyramid();
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

void b2f_lkpyr_pyramid_destroy(b2f_lkpyr_pyramid *p) { delete p; }

int b2f_lkpyr_build_pyramid(const b2f_image *img, int win_w, int win_h, int max_level, int with_derivatives, int pyr_border,
                            int deriv_border, b2f_lkpyr_pyramid *pyr, int *max_level_out, void *cuda_stream) {
    using namespace b2f;
    if (!pyr || win_w <= 2 || win_h <= 2 || max_level < 0) return B2F_BAD_ARG;
    int st = lk_image_ok(img);
    if (st != B2F_OK) return st;
    // BORDER_REFLECT_101 levels and BORDER_CONSTANT derivatives (BORDER_ISOLATED is implied): other modes are refused
    if ((pyr_border & ~16) != 4 || (deriv_border & ~16) != 0) return B2F_UNSUPPORTED_TYPE;
    const int levels = lk_levels(img->rows, img->cols, win_w, win_h, max_level);
    if (levels >= LK_MAX_LEVELS) return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(img->data, s);
    Ctx c;
    c.stream = s;
    if (pyr->layout(c, img->rows, img->cols, (img->type >> 3) + 1, win_w, win_h, levels + 1, with_derivatives ? 1 : 0) == B2F_OK)
        pyr->build(c, img);
    if (c.ok() && s == nullptr) c.check(cudaDeviceSynchronize());
    if (!c.ok()) {
        cudaGetLastError();
        return c.err == cudaErrorMemoryAllocation ? B2F_OUT_OF_MEMORY : B2F_CUDA_ERROR;
    }
    if (max_level_out) *max_level_out = levels;
    return B2F_OK;
}

int b2f_lkpyr_pyramid_info(const b2f_lkpyr_pyramid *p, int *levels, int *win_w, int *win_h, int *with_derivatives) {
    if (!p) return B2F_BAD_ARG;
    if (levels) *levels = p->levels;
    if (win_w) *win_w = p->win_w;
    if (win_h) *win_h = p->win_h;
    if (with_derivatives) *with_derivatives = p->derivs;
    return B2F_OK;
}

int b2f_lkpyr_pyramid_level(const b2f_lkpyr_pyramid *p, int level, int deriv, b2f_image *view) {
    if (!p || !view || level < 0 || level >= p->levels || (deriv && !p->derivs)) return B2F_BAD_ARG;
    const b2f_lkpyr_pyramid::Lvl &v = p->L[level];
    view->data = deriv ? static_cast<void *>(v.der) : static_cast<void *>(v.img);
    view->step = deriv ? v.dstep : v.istep;
    view->rows = v.rows + 2 * p->win_h;
    view->cols = v.cols + 2 * p->win_w;
    view->type = deriv ? (3 | ((2 * p->cn - 1) << 3)) : ((p->cn - 1) << 3);  // CV_16SC(2 cn) / CV_8UC(cn)
    return B2F_OK;
}

int b2f_lkpyr_calc(b2f_lkpyr *h, const b2f_image *prev_img, const b2f_lkpyr_pyramid *prev_pyr, const b2f_image *next_img,
                   const b2f_lkpyr_pyramid *next_pyr, const float *prev_pts, float *next_pts, unsigned char *status, float *err,
                   int n_points, void *cuda_stream) {
    using namespace b2f;
    if (!h || n_points < 0) return B2F_BAD_ARG;
    if ((prev_img != nullptr) == (prev_pyr != nullptr) || (next_img != nullptr) == (next_pyr != nullptr)) return B2F_BAD_ARG;
    const b2f_lkpyr_params &P = h->P;
    if (!lk_params_ok(P)) return B2F_BAD_ARG;
    int st;
    if (prev_img && (st = lk_image_ok(prev_img)) != B2F_OK) return st;
    if (next_img && (st = lk_image_ok(next_img)) != B2F_OK) return st;
    if (n_points == 0) return B2F_OK;
    if (!prev_pts || !next_pts || !status) return B2F_BAD_ARG;
    if (reinterpret_cast<uintptr_t>(prev_pts) % 8 || reinterpret_cast<uintptr_t>(next_pts) % 8 ||
        reinterpret_cast<uintptr_t>(err) % 4)
        return B2F_BAD_ARG;
    const int ww = P.win_width, wh = P.win_height;
    // calcOpticalFlowPyrLK's reconciliation: a pyramid caps maxLevel at its own level count, then each image is built
    // up to what is left (buildOpticalFlowPyramid may stop earlier)
    int max_level = P.max_level;
    for (const b2f_lkpyr_pyramid *p : {prev_pyr, next_pyr}) {
        if (!p) continue;
        if (p->levels < 1) return B2F_BAD_ARG;
        if (p->win_w < ww || p->win_h < wh) return B2F_BAD_ARG;  // CV_Assert(ofs.x >= winSize.width && ...)
        max_level = std::min(max_level, p->levels - 1);
    }
    if (prev_img) max_level = lk_levels(prev_img->rows, prev_img->cols, ww, wh, max_level);
    if (next_img) max_level = lk_levels(next_img->rows, next_img->cols, ww, wh, max_level);
    if (max_level >= LK_MAX_LEVELS) return B2F_BAD_ARG;
    const int prow = prev_img ? prev_img->rows : prev_pyr->rows, pcol = prev_img ? prev_img->cols : prev_pyr->cols;
    const int nrow = next_img ? next_img->rows : next_pyr->rows, ncol = next_img ? next_img->cols : next_pyr->cols;
    const int pcn = prev_img ? (prev_img->type >> 3) + 1 : prev_pyr->cn, ncn = next_img ? (next_img->type >> 3) + 1 : next_pyr->cn;
    if (prow != nrow || pcol != ncol) return B2F_SIZE_MISMATCH;
    if (pcn != ncn) return B2F_UNSUPPORTED_TYPE;

    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    const void *any = prev_img ? prev_img->data : next_img ? next_img->data : static_cast<const void *>(prev_pts);
    DeviceScope dev(any, s);
    if (!h->bind_device()) return B2F_BAD_ARG;
    Ctx c = h->make_ctx(s);
    h->stats.calls++;
    cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
    if (s && cudaStreamIsCapturing(s, &capturing) != cudaSuccess) cudaGetLastError();
    c.capturing = capturing != cudaStreamCaptureStatusNone;
    // order after the previous call when it ran on another stream (inside a caller's capture the caller orders)
    if (!c.capturing && h->done && h->last_stream != s) c.check(cudaStreamWaitEvent(s, h->done, 0));
    // workspace: the images' own pyramids, and derivatives for a prev pyramid built without them
    if (prev_img) h->own_prev.layout(c, prow, pcol, pcn, ww, wh, max_level + 1, 1);
    if (next_img && c.ok()) h->own_next.layout(c, nrow, ncol, ncn, ww, wh, max_level + 1, 0);
    const bool need_deriv = prev_pyr && !prev_pyr->derivs;
    if (need_deriv && c.ok()) h->own_deriv.layout(c, prow, pcol, pcn, prev_pyr->win_w, prev_pyr->win_h, max_level + 1, 1);
    if (!c.ok()) return h->finish(c, s);

    const b2f_lkpyr_pyramid &PI = prev_img ? h->own_prev : *prev_pyr;
    const b2f_lkpyr_pyramid &PJ = next_img ? h->own_next : *next_pyr;
    LkLevels Ls{};
    for (int l = 0; l <= max_level; ++l) {
        const auto &a = PI.L[l];
        const auto &b = PJ.L[l];
        const auto &d = need_deriv ? h->own_deriv.L[l] : a;
        const int dbw = need_deriv ? h->own_deriv.win_w : PI.win_w, dbh = need_deriv ? h->own_deriv.win_h : PI.win_h;
        if (a.rows != b.rows || a.cols != b.cols) return B2F_SIZE_MISMATCH;  // CV_Assert(prevPyr[l].size() == nextPyr[l].size())
        LkLevel &L = Ls.l[l];
        L.I = a.img + (size_t)PI.win_h * a.istep + (size_t)PI.win_w * pcn;
        L.dI = reinterpret_cast<const short *>(reinterpret_cast<const char *>(d.der) + (size_t)dbh * d.dstep) + (size_t)dbw * 2 * pcn;
        L.J = b.img + (size_t)PJ.win_h * b.istep + (size_t)PJ.win_w * pcn;
        L.istep = (int)a.istep;
        L.dstep = (int)(d.dstep / 2);
        L.jstep = (int)b.istep;
        L.rows = a.rows;
        L.cols = a.cols;
    }
    LkArgs A{};
    A.win_w = ww;
    A.win_h = wh;
    A.cn = pcn;
    A.max_level = max_level;
    A.max_count = (P.criteria_type & 1) ? std::min(std::max(P.max_count, 0), 100) : 30;
    double eps = (P.criteria_type & 2) ? std::min(std::max(P.epsilon, 0.), 10.) : 0.01;
    A.eps = eps * eps;
    A.flags = P.flags;
    A.min_eig = static_cast<float>(P.min_eig_threshold);

    b2f_lkpyr::Key key;
    key.prev = prev_img ? prev_img->data : nullptr;
    key.next = next_img ? next_img->data : nullptr;
    key.pstep = prev_img ? prev_img->step : 0;
    key.nstep = next_img ? next_img->step : 0;
    key.pp = prev_pts;
    key.np = next_pts;
    key.st = status;
    key.err = err;
    key.gen[0] = h->own_prev.generation;
    key.gen[1] = h->own_next.generation;
    key.rows = prow;
    key.cols = pcol;
    key.type = pcn;
    key.n = n_points;
    key.max_level = max_level;
    key.win_w = ww;
    key.win_h = wh;
    key.max_count = A.max_count;
    key.flags = A.flags;
    key.eps = A.eps;
    key.min_eig = A.min_eig;
    auto body = [&](Ctx &g) {
        if (prev_img) h->own_prev.build(g, prev_img);
        if (next_img) h->own_next.build(g, next_img);
        if (need_deriv) {
            // the prev pyramid's levels, seen through own_deriv's geometry (same sizes and border), feed k_lk_scharr
            for (int l = 0; l <= max_level; ++l) {
                const auto &v = h->own_deriv.L[l];
                const auto &src = prev_pyr->L[l];
                const dim3 blk(32, 8), grid(div_up(v.cols + 2 * prev_pyr->win_w, 32), div_up(v.rows + 2 * prev_pyr->win_h, 8));
                B2F_LAUNCH(g, CLS_DERIV, (double)(v.rows + 2 * prev_pyr->win_h) * (v.cols + 2 * prev_pyr->win_w) * pcn * 5.0,
                           k_lk_scharr, grid, blk, 0, src.img + (size_t)prev_pyr->win_h * src.istep + (size_t)prev_pyr->win_w * pcn,
                           src.istep, v.rows, v.cols, pcn, v.der, v.dstep, prev_pyr->win_w, prev_pyr->win_h);
            }
        }
        B2F_LAUNCH(g, CLS_TRACK, 0.0, k_lk_track, dim3(div_up(n_points, LK_BLOCK)), dim3(LK_BLOCK), 0, Ls, A,
                   reinterpret_cast<const float2 *>(prev_pts), reinterpret_cast<float2 *>(next_pts), status, err, n_points);
        // active path: one thread per point, every level in one launch (1); the levels it ran
        h->active_paths.assign(1, 1.0 + 256.0 * (max_level + 1));
    };
    if (!h->profiling && !c.capturing && h->knobs.use_graph && prev_img && next_img)
        h->graph.run(*h, c, s, key, body);
    else
        body(c);
    if (!c.capturing && c.ok()) {
        if (!h->done) c.check(cudaEventCreateWithFlags(&h->done, cudaEventDisableTiming));
        if (c.ok()) c.check(cudaEventRecord(h->done, s));
        h->last_stream = s;
    }
    return h->finish(c, s);
}

int b2f_lkpyr_last_cuda_error(const b2f_lkpyr *h) { return h ? h->last_cuda_error : 0; }

void b2f_lkpyr_destroy(b2f_lkpyr *h) { delete h; }

}  // extern "C"
