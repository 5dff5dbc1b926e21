// variational.cuh -- the cv::VariationalRefinement solver on the GPU, shared by the DeepFlow engine (deepflow.cu) and the
// DIS engine (dis.cu).  oracle/deepflow_model.py states what these kernels compute; both engines are compiled with
// -fmad=false so that every operator rounds once and the float model follows them bit for bit.
#pragma once

#include "common.cuh"

#include <algorithm>
#include <cmath>

namespace b2f {

namespace {

enum { CLS_SOR = 0, CLS_TERMS = 1, CLS_DERIV = 2, CLS_PYR = 3 };
constexpr float ZETA = 0.1f, EPSILON = 0.001f;

struct DFParams {
    float alpha2, delta2, gamma2, z2, e2, omega, omo;
};

// ---------------------------------------------------------------------------------------------
// pre-smoothing fused with the u8 / f32 -> float conversion (exact): 3x3 separable Gaussian, reflect-101 border;
// k0 x + k1 (l + r) along rows, then along columns.  Both frames per launch, read from the caller's pitched images.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect101(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return clampi(i, 0, n - 1);
}
template <typename T>
__device__ __forceinline__ float blur_row(const char *img, size_t step, int y, int x, int w, float k0, float k1) {
    const T *r = reinterpret_cast<const T *>(img + (size_t)y * step);
    return k0 * (float)r[x] + k1 * ((float)r[reflect101(x - 1, w)] + (float)r[reflect101(x + 1, w)]);
}
template <typename T>
__global__ void __launch_bounds__(256) k_df_blur(const char *s0, size_t step0, const char *s1, size_t step1, Plane d0, Plane d1,
                                                 int h, int w, float k0, float k1) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const char *s = blockIdx.z ? s1 : s0;
    const size_t st = blockIdx.z ? step1 : step0;
    const float c = blur_row<T>(s, st, y, x, w, k0, k1);
    const float a = blur_row<T>(s, st, reflect101(y - 1, h), x, w, k0, k1);
    const float b = blur_row<T>(s, st, reflect101(y + 1, h), x, w, k0, k1);
    (blockIdx.z ? d1 : d0).at(y, x) = k0 * c + k1 * (a + b);
}

// ---------------------------------------------------------------------------------------------
// cv::resize INTER_LINEAR (centre-aligned, modules/imgproc/src/resize.cpp): the source coordinate
// (d + 0.5) * (src / dst) - 0.5 in double, rounded to float, split into floor and fraction; below 0 or at the last
// source index the fraction is 0 and the index clamped.  Horizontal pass then vertical pass, each s0 (1 - f) + s1 f;
// times `mul` (the flow prolongation's 1 / 0.95f; 1 leaves the value unchanged).  Two planes per launch.  Unlike
// k_resize_linear in pyramid.cu (cv::cuda::resize, top-left aligned) this is the CPU resize the reference's driver
// calls.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void resize_coord(int d, double scale, int n, int &i0, int &i1, float &f) {
    const float fc = (float)(((double)d + 0.5) * scale - 0.5);
    int s = (int)floorf(fc);
    f = fc - (float)s;
    if (s < 0) { s = 0; f = 0.f; }
    if (s >= n - 1) { s = n - 1; f = 0.f; }
    i0 = s;
    i1 = min(s + 1, n - 1);
}
__global__ void __launch_bounds__(256) k_df_resize(Plane s0, Plane s1, int sh, int sw, Plane d0, Plane d1, int dh, int dw,
                                                   double sx, double sy, float mul, int apply_mul) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const Plane s = blockIdx.z ? s1 : s0;
    int x0, x1, y0, y1;
    float fx, fy;
    resize_coord(x, sx, sw, x0, x1, fx);
    resize_coord(y, sy, sh, y0, y1, fy);
    const float t0 = s.at(y0, x0) * (1.f - fx) + s.at(y0, x1) * fx;
    const float t1 = s.at(y1, x0) * (1.f - fx) + s.at(y1, x1) * fx;
    float r = t0 * (1.f - fy) + t1 * fy;
    if (apply_mul) r = r * mul;
    (blockIdx.z ? d1 : d0).at(y, x) = r;
}

// ---------------------------------------------------------------------------------------------
// per level, once: I1 warped by remap(INTER_LINEAR, BORDER_REPLICATE) -- coordinates rounded half to even to 1/32
// pixel, exact 1/32 weights, taps clamped -- then avg = 0.5 I0 + 0.5 warped I1 and Iz = warped I1 - I0
// ---------------------------------------------------------------------------------------------
struct WarpPlanes {
    Plane I0, I1, u, v, avg, Iz;
};
__global__ void __launch_bounds__(256) k_df_warp(WarpPlanes P, int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const float mx = (float)x + P.u.at(y, x), my = (float)y + P.v.at(y, x);
    const int X = __float2int_rn(mx * 32.f), Y = __float2int_rn(my * 32.f);
    const int x0 = X >> 5, y0 = Y >> 5;
    const float fx = (float)(X & 31) * (1.f / 32.f), fy = (float)(Y & 31) * (1.f / 32.f);
    const int xa = clampi(x0, 0, w - 1), xb = clampi(x0 + 1, 0, w - 1);
    const int ya = clampi(y0, 0, h - 1), yb = clampi(y0 + 1, 0, h - 1);
    const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
    const float wI = P.I1.at(ya, xa) * w00 + P.I1.at(ya, xb) * w01 + P.I1.at(yb, xa) * w10 + P.I1.at(yb, xb) * w11;
    const float i0 = P.I0.at(y, x);
    P.avg.at(y, x) = 0.5f * i0 + 0.5f * wI;
    P.Iz.at(y, x) = wI - i0;
}

// undivided central differences, replicated border: Ix, Iy of avg; Ixx, Ixy of Ix; Iyy of Iy; Ixz, Iyz of Iz
struct DerivPlanes {
    Plane avg, Iz, Ix, Iy, Ixx, Ixy, Iyy, Ixz, Iyz;
};
__device__ __forceinline__ float ddx(const Plane &p, int y, int x, int w) {
    return p.at(y, min(x + 1, w - 1)) - p.at(y, max(x - 1, 0));
}
__device__ __forceinline__ float ddy(const Plane &p, int y, int x, int h) {
    return p.at(min(y + 1, h - 1), x) - p.at(max(y - 1, 0), x);
}
__global__ void __launch_bounds__(256) k_df_deriv(DerivPlanes P, int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int xl = max(x - 1, 0), xr = min(x + 1, w - 1), yu = max(y - 1, 0), yd = min(y + 1, h - 1);
    P.Ix.at(y, x) = ddx(P.avg, y, x, w);
    P.Iy.at(y, x) = ddy(P.avg, y, x, h);
    P.Ixx.at(y, x) = ddx(P.avg, y, xr, w) - ddx(P.avg, y, xl, w);
    P.Ixy.at(y, x) = ddx(P.avg, yd, x, w) - ddx(P.avg, yu, x, w);
    P.Iyy.at(y, x) = ddy(P.avg, yd, x, h) - ddy(P.avg, yu, x, h);
    P.Ixz.at(y, x) = ddx(P.Iz, y, x, w);
    P.Iyz.at(y, x) = ddy(P.Iz, y, x, h);
}

// ---------------------------------------------------------------------------------------------
// one fixed-point step's linear system (oracle/deepflow_model.py system_terms)
// ---------------------------------------------------------------------------------------------
struct LevelPlanes {
    Plane Ix, Iy, Iz, Ixx, Ixy, Iyy, Ixz, Iyz;
    Plane u, v, du, dv;
    Plane a12, b1, b2, den_u, den_v, wr, wd;
};

// smoothness weight of pixel (x, y) from forward differences of (u + du, v + dv), zero difference at the far edge
__device__ __forceinline__ float smooth_weight(const LevelPlanes &P, int y, int x, int h, int w, const DFParams &k) {
    const int xr = min(x + 1, w - 1), yd = min(y + 1, h - 1);
    const float U = P.u.at(y, x) + P.du.at(y, x), V = P.v.at(y, x) + P.dv.at(y, x);
    const float ux = (P.u.at(y, xr) + P.du.at(y, xr)) - U, vx = (P.v.at(y, xr) + P.dv.at(y, xr)) - V;
    const float uy = (P.u.at(yd, x) + P.du.at(yd, x)) - U, vy = (P.v.at(yd, x) + P.dv.at(yd, x)) - V;
    return k.alpha2 / sqrtf(ux * ux + vx * vx + uy * uy + vy * vy + k.e2);
}

__device__ __forceinline__ void terms_cell(const LevelPlanes &P, int y, int x, int h, int w, const DFParams &k) {
    const float Ix = P.Ix.at(y, x), Iy = P.Iy.at(y, x), Iz = P.Iz.at(y, x);
    const float Ixx = P.Ixx.at(y, x), Ixy = P.Ixy.at(y, x), Iyy = P.Iyy.at(y, x);
    const float Ixz = P.Ixz.at(y, x), Iyz = P.Iyz.at(y, x);
    const float du = P.du.at(y, x), dv = P.dv.at(y, x);
    // colour constancy
    const float n = Ix * Ix + Iy * Iy + k.z2;
    const float q = Iz + Ix * du + Iy * dv;
    const float wt = k.delta2 / sqrtf(q * q / n + k.e2) / n;
    float a11 = wt * (Ix * Ix) + k.z2;
    float a12 = wt * (Ix * Iy);
    float a22 = wt * (Iy * Iy) + k.z2;
    float b1 = -(wt * (Iz * Ix));
    float b2 = -(wt * (Iz * Iy));
    // gradient constancy
    const float n1 = Ixx * Ixx + Ixy * Ixy + k.z2;
    const float n2 = Iyy * Iyy + Ixy * Ixy + k.z2;
    const float qx = Ixz + Ixx * du + Ixy * dv;
    const float qy = Iyz + Ixy * du + Iyy * dv;
    const float wg = k.gamma2 / sqrtf(qx * qx / n1 + qy * qy / n2 + k.e2);
    a11 = a11 + wg * (Ixx * Ixx / n1 + Ixy * Ixy / n2);
    a12 = a12 + wg * (Ixx * Ixy / n1 + Ixy * Iyy / n2);
    a22 = a22 + wg * (Ixy * Ixy / n1 + Iyy * Iyy / n2);
    b1 = b1 - wg * (Ixx * Ixz / n1 + Ixy * Iyz / n2);
    b2 = b2 - wg * (Ixy * Ixz / n1 + Iyy * Iyz / n2);
    // smoothness: edge weights to the right / below (this pixel's weight) and to the left / above (the neighbour's)
    const float s = smooth_weight(P, y, x, h, w, k);
    const float wr = x < w - 1 ? s : 0.f, wd = y < h - 1 ? s : 0.f;
    const float wl = x > 0 ? smooth_weight(P, y, x - 1, h, w, k) : 0.f;
    const float wu = y > 0 ? smooth_weight(P, y - 1, x, h, w, k) : 0.f;
    const int xr = min(x + 1, w - 1), xl = max(x - 1, 0), yd = min(y + 1, h - 1), yu = max(y - 1, 0);
    const float u = P.u.at(y, x), v = P.v.at(y, x);
    b1 = b1 + (wr * (P.u.at(y, xr) - u) + wl * (P.u.at(y, xl) - u) + wd * (P.u.at(yd, x) - u) + wu * (P.u.at(yu, x) - u));
    b2 = b2 + (wr * (P.v.at(y, xr) - v) + wl * (P.v.at(y, xl) - v) + wd * (P.v.at(yd, x) - v) + wu * (P.v.at(yu, x) - v));
    const float S = wr + wl + wd + wu;
    P.a12.at(y, x) = a12;
    P.b1.at(y, x) = b1;
    P.b2.at(y, x) = b2;
    P.den_u.at(y, x) = a11 + S;
    P.den_v.at(y, x) = a22 + S;
    P.wr.at(y, x) = wr;
    P.wd.at(y, x) = wd;
}

__global__ void __launch_bounds__(256) k_df_terms(LevelPlanes P, int h, int w, DFParams k) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    terms_cell(P, y, x, h, w, k);
}

// ---------------------------------------------------------------------------------------------
// One SOR cell update, shared by both solver kernels (same expression order as deepflow_model.sor):
//   du' = (1 - omega) du + omega ((b1 + sum w du_nb) - a12 dv) / den_u,  then dv' with the new du.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void sor_cell(float wr, float wl, float wd, float wu, float a12, float b1, float b2, float den_u,
                                         float den_v, float dur, float dul, float dud, float duu, float dvr, float dvl,
                                         float dvd, float dvu, const DFParams &k, float &du, float &dv) {
    const float su = wr * dur + wl * dul + wd * dud + wu * duu;
    du = k.omo * du + k.omega * (b1 + su - a12 * dv) / den_u;
    const float sv = wr * dvr + wl * dvl + wd * dvd + wu * dvu;
    dv = k.omo * dv + k.omega * (b2 + sv - a12 * du) / den_v;
}

// ---------------------------------------------------------------------------------------------
// Region solver: `iters` full red-black iterations per launch on a 64x64 region held in shared memory.  Each half
// sweep consumes one halo cell per side, so with a halo of 2 * iters the centre (64 - 4 iters)^2 tile is exact; a
// colour's update reads only the other colour, so updating in place equals a sweep over the whole level.  Launches
// ping-pong (du, dv) between two plane pairs: a CTA reads its halo from cells other CTAs write.  Cells outside the
// image carry zero weights and are never updated.
// ---------------------------------------------------------------------------------------------
constexpr int SR = 64, SOR_THREADS = 512, SOR_PLANES = 9;

__global__ void __launch_bounds__(SOR_THREADS, 1)
    k_df_sor(LevelPlanes P, Plane du_out, Plane dv_out, int h, int w, DFParams k, int iters, int halo, int tile) {
    extern __shared__ float sm[];
    float *s_du = sm, *s_dv = sm + SR * SR, *s_a12 = sm + 2 * SR * SR, *s_b1 = sm + 3 * SR * SR, *s_b2 = sm + 4 * SR * SR;
    float *s_du_den = sm + 5 * SR * SR, *s_dv_den = sm + 6 * SR * SR, *s_wr = sm + 7 * SR * SR, *s_wd = sm + 8 * SR * SR;
    const int tid = threadIdx.x;
    const int gx0 = blockIdx.x * tile - halo, gy0 = blockIdx.y * tile - halo;
    for (int idx = tid; idx < SR * SR; idx += SOR_THREADS) {
        const int ry = idx >> 6, rx = idx & 63, gy = gy0 + ry, gx = gx0 + rx;
        const bool in = gx >= 0 && gy >= 0 && gx < w && gy < h;
        s_du[idx] = in ? P.du.at(gy, gx) : 0.f;
        s_dv[idx] = in ? P.dv.at(gy, gx) : 0.f;
        s_a12[idx] = in ? P.a12.at(gy, gx) : 0.f;
        s_b1[idx] = in ? P.b1.at(gy, gx) : 0.f;
        s_b2[idx] = in ? P.b2.at(gy, gx) : 0.f;
        s_du_den[idx] = in ? P.den_u.at(gy, gx) : 0.f;
        s_dv_den[idx] = in ? P.den_v.at(gy, gx) : 0.f;
        s_wr[idx] = in ? P.wr.at(gy, gx) : 0.f;
        s_wd[idx] = in ? P.wd.at(gy, gx) : 0.f;
    }
    __syncthreads();
    for (int sweep = 0; sweep < 2 * iters; ++sweep) {
        const int colour = sweep & 1;  // cells with even x + y first
        for (int c = tid; c < SR * SR / 2; c += SOR_THREADS) {
            const int ry = c >> 5;
            const int rx = ((c & 31) << 1) + ((ry + gy0 + gx0 + colour) & 1);
            const int gy = gy0 + ry, gx = gx0 + rx;
            if (gx < 0 || gy < 0 || gx >= w || gy >= h) continue;
            // region-edge cells read clamped region neighbours: stale, but they lie in the halo
            const int idx = ry * SR + rx;
            const int il = rx > 0 ? idx - 1 : idx, ir = rx < SR - 1 ? idx + 1 : idx;
            const int iu = ry > 0 ? idx - SR : idx, id = ry < SR - 1 ? idx + SR : idx;
            const float wl = rx > 0 ? s_wr[il] : 0.f, wu = ry > 0 ? s_wd[iu] : 0.f;
            float du = s_du[idx], dv = s_dv[idx];
            sor_cell(s_wr[idx], wl, s_wd[idx], wu, s_a12[idx], s_b1[idx], s_b2[idx], s_du_den[idx], s_dv_den[idx], s_du[ir],
                     s_du[il], s_du[id], s_du[iu], s_dv[ir], s_dv[il], s_dv[id], s_dv[iu], k, du, dv);
            s_du[idx] = du;
            s_dv[idx] = dv;
        }
        __syncthreads();
    }
    for (int idx = tid; idx < tile * tile; idx += SOR_THREADS) {
        const int ty = idx / tile, tx = idx - ty * tile;
        const int gy = gy0 + halo + ty, gx = gx0 + halo + tx;
        if (gx < w && gy < h) {
            du_out.at(gy, gx) = s_du[(halo + ty) * SR + halo + tx];
            dv_out.at(gy, gx) = s_dv[(halo + ty) * SR + halo + tx];
        }
    }
}

// A level that fits one 64x64 region: every fixed-point step (system terms + all SOR iterations) and u += du in one
// CTA, in global memory (writes of a CTA are visible to it after a barrier).  Same device functions as the kernels
// above: bit-identical to them.
constexpr int SMALL_THREADS = 1024;
__global__ void __launch_bounds__(SMALL_THREADS, 1)
    k_df_level_small(LevelPlanes P, int h, int w, DFParams k, int fp_iters, int sor_iters) {
    const int tid = threadIdx.x, n = h * w;
    for (int i = tid; i < n; i += SMALL_THREADS) {
        const int y = i / w, x = i - y * w;
        P.du.at(y, x) = 0.f;
        P.dv.at(y, x) = 0.f;
    }
    __syncthreads();
    for (int f = 0; f < fp_iters; ++f) {
        for (int i = tid; i < n; i += SMALL_THREADS) {
            const int y = i / w, x = i - y * w;
            terms_cell(P, y, x, h, w, k);
        }
        __syncthreads();
        for (int sweep = 0; sweep < 2 * sor_iters; ++sweep) {
            const int colour = sweep & 1;
            const int half = (w + 1) >> 1;  // slots per row for one colour
            for (int c = tid; c < h * half; c += SMALL_THREADS) {
                const int y = c / half, x = ((c - y * half) << 1) + ((y + colour) & 1);
                if (y >= h || x >= w) continue;
                const int xl = max(x - 1, 0), xr = min(x + 1, w - 1), yu = max(y - 1, 0), yd = min(y + 1, h - 1);
                const float wl = x > 0 ? P.wr.at(y, xl) : 0.f, wu = y > 0 ? P.wd.at(yu, x) : 0.f;
                float du = P.du.at(y, x), dv = P.dv.at(y, x);
                sor_cell(P.wr.at(y, x), wl, P.wd.at(y, x), wu, P.a12.at(y, x), P.b1.at(y, x), P.b2.at(y, x),
                         P.den_u.at(y, x), P.den_v.at(y, x), P.du.at(y, xr), P.du.at(y, xl), P.du.at(yd, x),
                         P.du.at(yu, x), P.dv.at(y, xr), P.dv.at(y, xl), P.dv.at(yd, x), P.dv.at(yu, x), k, du, dv);
                P.du.at(y, x) = du;
                P.dv.at(y, x) = dv;
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < n; i += SMALL_THREADS) {
        const int y = i / w, x = i - y * w;
        P.u.at(y, x) = P.u.at(y, x) + P.du.at(y, x);
        P.v.at(y, x) = P.v.at(y, x) + P.dv.at(y, x);
    }
}

// u += du, v += dv
__global__ void __launch_bounds__(256) k_df_add(Plane u, Plane v, Plane du, Plane dv, int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    u.at(y, x) = u.at(y, x) + du.at(y, x);
    v.at(y, x) = v.at(y, x) + dv.at(y, x);
}
// SOR iterations per solver launch on an h x w level.  More iterations per launch = fewer launches but a wider halo
// (smaller tile, more CTAs).  Cost model in microseconds, per wave of one CTA per SM: region fill ~3, half sweep
// ~0.35, launch gap ~2 (the Brox solver's model; the DeepFlow cell update is the same stencil).
inline int variational_iters_per_launch(int sor_iterations, int h, int w, int num_sms) {
    const int n = sor_iterations;
    if (w <= SR && h <= SR) return n;
    int best_it = 1;
    double best = 1e30;
    for (int cand = 1; cand <= 12 && cand <= n; ++cand) {
        const int t = SR - 4 * cand;
        if (t < 8) break;
        const int launches = div_up(n, cand);
        const double waves = std::ceil((double)div_up(w, t) * div_up(h, t) / (double)num_sms);
        const double cost = launches * (waves * (3.0 + 0.7 * cand) + 2.0);
        if (cost < best) {
            best = cost;
            best_it = cand;
        }
    }
    return best_it;
}

// One VariationalRefinement::calcUV call on an h x w level: T.u, T.v += the increment.  I0 / I1 are the level's
// frames, `avg` a spare plane (dead once the derivatives are written, so it may alias T.a12), (dun, dvn) the solver's
// ping-pong pair.  `it` is variational_iters_per_launch for the level.  Kernel classes: cls_sor, cls_terms, cls_deriv
// and cls_add (u += du).
inline void variational_level(Ctx &c, LevelPlanes T, Plane I0, Plane I1, Plane avg, Plane dun, Plane dvn, int h, int w,
                              const DFParams &k, int fp_iters, int sor_iters, int it, int cls_sor, int cls_terms,
                              int cls_deriv, int cls_add) {
    const dim3 block(32, 8);
    const size_t sor_smem = sizeof(float) * SOR_PLANES * SR * SR;
    const double npx = (double)h * w;
    const dim3 grid(div_up(w, 32), div_up(h, 8));
    WarpPlanes W{I0, I1, T.u, T.v, avg, T.Iz};
    B2F_LAUNCH(c, cls_deriv, 32.0 * npx, k_df_warp, grid, block, 0, W, h, w);
    DerivPlanes D{W.avg, T.Iz, T.Ix, T.Iy, T.Ixx, T.Ixy, T.Iyy, T.Ixz, T.Iyz};
    B2F_LAUNCH(c, cls_deriv, 36.0 * npx, k_df_deriv, grid, block, 0, D, h, w);
    if (w <= SR && h <= SR) {
        // terms 88 B/px per step; the SOR's share as for the region solver
        B2F_LAUNCH(c, cls_sor, (88.0 + 44.0 * sor_iters) * npx * fp_iters + 24.0 * npx, k_df_level_small, dim3(1),
                   dim3(SMALL_THREADS), 0, T, h, w, k, fp_iters, sor_iters);
        if (c.ok()) c.stats->iterations_run += sor_iters * fp_iters;
        return;
    }
    fill_plane(c, T.du, h, w, 0.f);
    fill_plane(c, T.dv, h, w, 0.f);
    for (int f = 0; f < fp_iters; ++f) {
        B2F_LAUNCH(c, cls_terms, 88.0 * npx, k_df_terms, grid, block, 0, T, h, w, k);
        int left = sor_iters;
        Plane cdu = T.du, cdv = T.dv, ndu = dun, ndv = dvn;
        while (left > 0) {
            const int n = std::min(left, it);
            const int halo = 2 * n, tile = SR - 2 * halo;
            LevelPlanes Q = T;
            Q.du = cdu;
            Q.dv = cdv;
            B2F_LAUNCH(c, cls_sor, 44.0 * npx * n, k_df_sor, dim3(div_up(w, tile), div_up(h, tile)), dim3(SOR_THREADS),
                       sor_smem, Q, ndu, ndv, h, w, k, n, halo, tile);
            std::swap(cdu, ndu);
            std::swap(cdv, ndv);
            left -= n;
            c.stats->iterations_run += n;
        }
        if (cdu.p != T.du.p) {  // odd number of launches: the result sits in the spare pair
            std::swap(T.du, dun);
            std::swap(T.dv, dvn);
        }
    }
    B2F_LAUNCH(c, cls_add, 24.0 * npx, k_df_add, grid, block, 0, T.u, T.v, T.du, T.dv, h, w);
}

}  // namespace

}  // namespace b2f
