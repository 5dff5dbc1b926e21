// brox.cu -- cv::cuda::BroxOpticalFlow re-implemented for sm_90a.
//
// Reference being replaced:
//   modules/cudaoptflow/src/brox.cpp:129-188                       (BroxOpticalFlowImpl::calc shim)
//   modules/cudalegacy/src/cuda/NCVBroxOpticalFlow.cu:188-554,598-985 (solver)         [NB]
//   modules/cudalegacy/src/cuda/NPP_staging.cu:1433-1501,2072-2231     (filters, resizers) [NS]
//
// Differences by design:
//  * one stream, no host synchronisation, whole solve captured in a CUDA graph (the reference issues
//    >= 6 cudaStreamSynchronize per call plus one per pyramid level and runs its filters/resizers on
//    the global NPP stream regardless of the caller's, NS:60-75);
//  * no texture objects: bilinear sampling with mirror addressing is done in software with exact
//    float32 weights (the reference's hardware filtering uses 9-bit fixed-point weights);
//  * prepare_sor stage 1 + stage 2 fused (the neighbours' diffusivities are recomputed instead of
//    making a second pass), u += du fused into the prolongation.
//
// Kernel classes: 0 sor (red/black half sweep, 52 B/px algorithmic per pair of half sweeps),
// 1 prepare (104 B/px), 2 derivatives, 3 pyramid (supersample / bicubic prolongation / add).
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace b2f {

namespace {

enum { CLS_SOR = 0, CLS_PREP = 1, CLS_DERIV = 2, CLS_PYR = 3 };
constexpr float EPS2 = 1e-6f;  // NB:78

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int mirror_filter(int i, int n) {  // NS:1433-1447 (asymmetric low side)
    if (i < 0) i = 1 - i;
    if (i >= n) i = n + n - i - 1;
    return clampi(i, 0, n - 1);
}
__device__ __forceinline__ int mirror_tex(int i, int n) {  // cudaAddressModeMirror on texel indices
    const int p = 2 * n;
    i %= p;
    if (i < 0) i += p;
    return i >= n ? p - 1 - i : i;
}
__device__ __forceinline__ int mirror_load(int i, int n) {  // load_array_element, NB:243-246
    i = max(i, -i - 1);
    i = min(i, n - i + n - 1);
    return clampi(i, 0, n - 1);
}

// Rounding: the Brox kernels spell out every multiply-add rounding with __fmaf_rn / __fmul_rn / __fadd_rn, exactly
// where nvcc -O3 fused or did not fuse the plain expressions (oracle/brox_model.py restates them one for one).  Plain
// operators remain only where no contraction is possible (a sum of loads, a product that feeds no addition).

// Normalised-coordinate, linear, mirror-addressed fetch (software replacement of the texture unit).
__device__ __forceinline__ float tex_bilinear(const Plane &P, int h, int w, float xn, float yn) {
    const float xb = __fmaf_rn(xn, (float)w, -0.5f), yb = __fmaf_rn(yn, (float)h, -0.5f);
    const float fx0 = floorf(xb), fy0 = floorf(yb);
    const float ax = __fsub_rn(xb, fx0), ay = __fsub_rn(yb, fy0);
    const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
    // keep the integer conversion safe for wild flows; mirror addressing is periodic anyway
    const int x0 = (int)fminf(fmaxf(fx0, -1.0e6f), 1.0e6f), y0 = (int)fminf(fmaxf(fy0, -1.0e6f), 1.0e6f);
    const int xa = mirror_tex(x0, w), xc = mirror_tex(x0 + 1, w);
    const int ya = mirror_tex(y0, h), yc = mirror_tex(y0 + 1, h);
    const float top = __fmaf_rn(bx, __ldg(&P.at(ya, xa)), __fmul_rn(ax, __ldg(&P.at(ya, xc))));
    const float bot = __fmaf_rn(bx, __ldg(&P.at(yc, xa)), __fmul_rn(ax, __ldg(&P.at(yc, xc))));
    return __fmaf_rn(by, top, __fmul_rn(ay, bot));
}

// ---------------------------------------------------------------------------------------------
// pyramid: supersample restriction (NS:2073-2149), both frames per launch
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float ss_line(const float *row, int sw, float xmin, float xmax, int ixmin, int ixmax,
                                         float fxmin, float cxmax) {
    const float w0 = __fadd_rn(__fsub_rn(1.0f, xmin), fxmin), w1 = __fsub_rn(cxmax, xmax);
    float wsum = w0;
    float sum = __fmul_rn(__ldg(row + ixmin), w0);
    int sp = ixmin + 1;
    for (int ix = ixmin + 1; ix < ixmax; ++ix) {
        sum = __fadd_rn(sum, __ldg(row + min(sp, sw - 1)));
        sp++;
        wsum = __fadd_rn(wsum, 1.0f);
    }
    sum = __fmaf_rn(w1, __ldg(row + min(sp, sw - 1)), sum);
    wsum = __fadd_rn(wsum, w1);
    return __fdiv_rn(sum, wsum);
}

__global__ void __launch_bounds__(256) k_brox_supersample(Plane s0, Plane s1, int sh, int sw, Plane d0, Plane d1, int dh,
                                                          int dw, float scale) {
    const int ix = blockIdx.x * blockDim.x + threadIdx.x;
    const int iy = blockIdx.y * blockDim.y + threadIdx.y;
    if (ix >= dw || iy >= dh) return;
    const Plane src = blockIdx.z ? s1 : s0;
    const float rw = (float)sw, rh = (float)sh;
    // x = scale * ix is never rounded on its own: both bounds fuse the product
    const float fx = (float)ix, fy = (float)iy;
    const float xBegin = fmaxf(__fmaf_rn(fx, scale, -scale), 0.0f), xEnd = fminf(__fmaf_rn(fx, scale, scale), __fsub_rn(rw, 1.0f));
    const float yBegin = fmaxf(__fmaf_rn(fy, scale, -scale), 0.0f), yEnd = fminf(__fmaf_rn(fy, scale, scale), __fsub_rn(rh, 1.0f));
    const float fxb = floorf(xBegin), cxe = ceilf(xEnd);
    const int iXBegin = (int)fxb, iXEnd = (int)cxe;
    const float fyb = floorf(yBegin), cye = ceilf(yEnd);
    const int iYBegin = (int)fyb, iYEnd = (int)cye;
    int ry = iYBegin;
    const float w0 = __fadd_rn(__fsub_rn(1.0f, yBegin), fyb), w1 = __fsub_rn(cye, yEnd);
    float wsum = w0;
    float sum = __fmul_rn(ss_line(src.row(ry), sw, xBegin, xEnd, iXBegin, iXEnd, fxb, cxe), w0);
    ry++;
    for (int yy = iYBegin + 1; yy < iYEnd; ++yy) {
        sum = __fadd_rn(sum, ss_line(src.row(min(ry, sh - 1)), sw, xBegin, xEnd, iXBegin, iXEnd, fxb, cxe));
        ry++;
        wsum = __fadd_rn(wsum, 1.0f);
    }
    sum = __fmaf_rn(w1, ss_line(src.row(min(ry, sh - 1)), sw, xBegin, xEnd, iXBegin, iXEnd, fxb, cxe), sum);
    wsum = __fadd_rn(wsum, w1);
    (blockIdx.z ? d1 : d0).at(iy, ix) = __fdiv_rn(sum, wsum);
}

// ---------------------------------------------------------------------------------------------
// derivative bank: {1,-8,0,8,-1}/12 with the reference's mirror rule (NS:1449-1501; NB:843-868)
// pass 1: Ix0, Iy0 (from I0), Ix, Iy (from I1);  pass 2: Ixx = dx(Ix), Iyy = dy(Iy), Ixy = dx(Iy)
// The taps are left to nvcc: a product by +-1, +-8 or 0 is exact, so fusing it into the sum cannot change a bit.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float d5_row(const Plane &P, int y, int x, int w) {
    float sum = 0.0f;
    sum += __ldg(&P.at(y, mirror_filter(x - 2, w))) * 1.0f;
    sum += __ldg(&P.at(y, mirror_filter(x - 1, w))) * -8.0f;
    sum += __ldg(&P.at(y, mirror_filter(x, w))) * 0.0f;
    sum += __ldg(&P.at(y, mirror_filter(x + 1, w))) * 8.0f;
    sum += __ldg(&P.at(y, mirror_filter(x + 2, w))) * -1.0f;
    return sum * (1.0f / 12.0f);
}
__device__ __forceinline__ float d5_col(const Plane &P, int y, int x, int h) {
    float sum = 0.0f;
    sum += __ldg(&P.at(mirror_filter(y - 2, h), x)) * 1.0f;
    sum += __ldg(&P.at(mirror_filter(y - 1, h), x)) * -8.0f;
    sum += __ldg(&P.at(mirror_filter(y, h), x)) * 0.0f;
    sum += __ldg(&P.at(mirror_filter(y + 1, h), x)) * 8.0f;
    sum += __ldg(&P.at(mirror_filter(y + 2, h), x)) * -1.0f;
    return sum * (1.0f / 12.0f);
}

__global__ void __launch_bounds__(256) k_brox_deriv1(Plane I0, Plane I1, Plane Ix0, Plane Iy0, Plane Ix, Plane Iy,
                                                     int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    Ix0.at(y, x) = d5_row(I0, y, x, w);
    Iy0.at(y, x) = d5_col(I0, y, x, h);
    Ix.at(y, x) = d5_row(I1, y, x, w);
    Iy.at(y, x) = d5_col(I1, y, x, h);
}

__global__ void __launch_bounds__(256) k_brox_deriv2(Plane Ix, Plane Iy, Plane Ixx, Plane Iyy, Plane Ixy, int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    Ixx.at(y, x) = d5_row(Ix, y, x, w);
    Iyy.at(y, x) = d5_col(Iy, y, x, h);
    Ixy.at(y, x) = d5_row(Iy, y, x, w);
}

// ---------------------------------------------------------------------------------------------
// prepare_sor: stage 1 (NB:340-406) + stage 2 (NB:416-473) fused
// ---------------------------------------------------------------------------------------------
struct BroxLevelPlanes {
    Plane I0, I1, Ix, Ixx, Ix0, Iy, Iyy, Iy0, Ixy;
    Plane u, v, du, dv;
    Plane sx, sy, inv_u, inv_v, num_dudv, num_u, num_v;
    // warped image terms, constant over the inner iterations of a level (they depend on (u, v) only)
    Plane wIz, wIx, wIxz, wIxy, wIxx, wIy, wIyz, wIyy;
};

// Shared-memory tile of (u, du, v, dv) with a 1-cell halo, mirror-addressed like load_array_element (NB:238-319).
constexpr int PB_X = 32, PB_Y = 8;
constexpr int PT_W = PB_X + 2, PT_H = PB_Y + 2;
struct PrepTile {
    float u[PT_H][PT_W], du[PT_H][PT_W], v[PT_H][PT_W], dv[PT_H][PT_W];
};
// 0.5 / sqrt(u_x^2 + v_x^2 + u_y^2 + v_y^2 + EPS2); the differences themselves are plain sums of loads
__device__ __forceinline__ float brox_diffusivity(float u_x, float v_x, float u_y, float v_y) {
    float s = __fmaf_rn(u_x, u_x, __fmul_rn(v_x, v_x));
    s = __fmaf_rn(u_y, u_y, s);
    s = __fmaf_rn(v_y, v_y, s);
    return __fdiv_rn(0.5f, __fsqrt_rn(__fadd_rn(s, EPS2)));
}
// diffusivity between (i,j) and (i-1,j)  (NB:188-204); (ty, tx) = tile coordinates of (j, i)
__device__ __forceinline__ float brox_sx(const PrepTile &T, int ty, int tx) {
    const float u_x = T.u[ty][tx] + T.du[ty][tx] - T.u[ty][tx - 1] - T.du[ty][tx - 1];
    const float v_x = T.v[ty][tx] + T.dv[ty][tx] - T.v[ty][tx - 1] - T.dv[ty][tx - 1];
    const float u_y = 0.25f * (T.u[ty + 1][tx] + T.du[ty + 1][tx] + T.u[ty + 1][tx - 1] + T.du[ty + 1][tx - 1] -
                               T.u[ty - 1][tx] - T.du[ty - 1][tx] - T.u[ty - 1][tx - 1] - T.du[ty - 1][tx - 1]);
    const float v_y = 0.25f * (T.v[ty + 1][tx] + T.dv[ty + 1][tx] + T.v[ty + 1][tx - 1] + T.dv[ty + 1][tx - 1] -
                               T.v[ty - 1][tx] - T.dv[ty - 1][tx] - T.v[ty - 1][tx - 1] - T.dv[ty - 1][tx - 1]);
    return brox_diffusivity(u_x, v_x, u_y, v_y);
}
// diffusivity between (i,j) and (i,j-1)  (NB:216-227)
__device__ __forceinline__ float brox_sy(const PrepTile &T, int ty, int tx) {
    const float u_y = T.u[ty][tx] + T.du[ty][tx] - T.u[ty - 1][tx] - T.du[ty - 1][tx];
    const float v_y = T.v[ty][tx] + T.dv[ty][tx] - T.v[ty - 1][tx] - T.dv[ty - 1][tx];
    const float u_x = 0.25f * (T.u[ty][tx + 1] + T.u[ty - 1][tx + 1] + T.du[ty][tx + 1] + T.du[ty - 1][tx + 1] -
                               T.u[ty][tx - 1] - T.u[ty - 1][tx - 1] - T.du[ty][tx - 1] - T.du[ty - 1][tx - 1]);
    const float v_x = 0.25f * (T.v[ty][tx + 1] + T.v[ty - 1][tx + 1] + T.dv[ty][tx + 1] + T.dv[ty - 1][tx + 1] -
                               T.v[ty][tx - 1] - T.v[ty - 1][tx - 1] - T.dv[ty][tx - 1] - T.dv[ty - 1][tx - 1]);
    return brox_diffusivity(u_x, v_x, u_y, v_y);
}

// The texture fetches of prepare_sor_stage_1 (NB:352-383): I1 and its derivatives sampled at the warped
// position ((x + u) / w, (y + v) / h), I0 and its derivatives at the pixel centre.  (u, v) do not change
// during the inner iterations of a level -- only (du, dv) do -- so the reference's 9 bilinear fetches per
// pixel per inner iteration are evaluated once per level here and re-read as 8 coalesced planes.
__global__ void __launch_bounds__(256) k_brox_warp_terms(BroxLevelPlanes P, int h, int w) {
    const int ig = blockIdx.x * blockDim.x + threadIdx.x;
    const int jg = blockIdx.y * blockDim.y + threadIdx.y;
    if (ig >= w || jg >= h) return;
    float x = (float)ig + 0.5f, y = (float)jg + 0.5f;
    const float uu = P.u.at(jg, ig), vv = P.v.at(jg, ig);
    const float wx = (x + uu) / (float)w, wy = (y + vv) / (float)h;
    x /= (float)w;
    y /= (float)h;
    const float Ix = tex_bilinear(P.Ix, h, w, wx, wy);
    const float Iy = tex_bilinear(P.Iy, h, w, wx, wy);
    P.wIz.at(jg, ig) = tex_bilinear(P.I1, h, w, wx, wy) - tex_bilinear(P.I0, h, w, x, y);
    P.wIx.at(jg, ig) = Ix;
    P.wIxz.at(jg, ig) = Ix - tex_bilinear(P.Ix0, h, w, x, y);
    P.wIxy.at(jg, ig) = tex_bilinear(P.Ixy, h, w, wx, wy);
    P.wIxx.at(jg, ig) = tex_bilinear(P.Ixx, h, w, wx, wy);
    P.wIy.at(jg, ig) = Iy;
    P.wIyz.at(jg, ig) = Iy - tex_bilinear(P.Iy0, h, w, x, y);
    P.wIyy.at(jg, ig) = tex_bilinear(P.Iyy, h, w, wx, wy);
}

// prepare_sor_stage_1 + stage_2 fused (NB:340-473).  The smoothness diffusivities are computed once per cell
// edge from a shared tile (each is needed by the two cells it separates) instead of four 24-load evaluations
// per pixel; the data term samples the warped image and its derivatives in software.
// One 32 x 8 chunk worked by 256 threads (tid = ty * 32 + tx); every thread of the CTA must call it (two barriers),
// `active` = the chunk exists.  CG: read what other CTAs of the SAME launch wrote (du, dv) through L2 (ld.global.cg) --
// the cooperative level kernel below runs many inner iterations in one launch, and L1 is not coherent.
template <bool CG>
__device__ __forceinline__ float brox_ld(const Plane &p, int y, int x) {
    return CG ? __ldcg(&p.at(y, x)) : p.at(y, x);
}
struct PrepShared {
    PrepTile T;
    float sx[PB_Y][PB_X + 1];   // sx at tile columns 0..32
    float sy[PB_Y + 1][PB_X];   // sy at tile rows 0..8
};
// EXACT_RSQ (aux_path 1, a test knob): the data term's reciprocal square root correctly rounded (__frsqrt_rn) instead
// of rsqrtf (MUFU.RSQ, up to 2 ulp, bits unspecified), so that a float model can follow the engine bit for bit.
template <bool CG, bool EXACT_RSQ>
__device__ __forceinline__ void brox_prepare_chunk(const BroxLevelPlanes &P, int h, int w, float alpha, float gamma, int gx0,
                                                   int gy0, int tid, PrepShared &S, bool active) {
    PrepTile &T = S.T;
    const int tx = tid & (PB_X - 1), ty = tid / PB_X;
    if (active) {
        for (int t = tid; t < PT_W * PT_H; t += PB_X * PB_Y) {
            const int ry = t / PT_W, rx = t - ry * PT_W;
            const int y = mirror_load(gy0 - 1 + ry, h), x = mirror_load(gx0 - 1 + rx, w);
            T.u[ry][rx] = P.u.at(y, x);
            T.du[ry][rx] = brox_ld<CG>(P.du, y, x);
            T.v[ry][rx] = P.v.at(y, x);
            T.dv[ry][rx] = brox_ld<CG>(P.dv, y, x);
        }
    }
    __syncthreads();
    constexpr int N_SX = PB_Y * (PB_X + 1), N_SY = (PB_Y + 1) * PB_X;
    if (active) {
        for (int t = tid; t < N_SX + N_SY; t += PB_X * PB_Y) {
            if (t < N_SX) {
                const int ry = t / (PB_X + 1), rx = t - ry * (PB_X + 1);
                const int gy = gy0 + ry, gx = gx0 + rx;
                // sx = 0 at i = 0 (NB:396) and beyond the image (stage 2 treats it as zero, NB:440-452)
                S.sx[ry][rx] = (gx == 0 || gx >= w || gy >= h) ? 0.f : brox_sx(T, ry + 1, rx + 1);
            } else {
                const int q = t - N_SX;
                const int ry = q / PB_X, rx = q - ry * PB_X;
                const int gy = gy0 + ry, gx = gx0 + rx;
                S.sy[ry][rx] = (gy == 0 || gy >= h || gx >= w) ? 0.f : brox_sy(T, ry + 1, rx + 1);
            }
        }
    }
    __syncthreads();

    const int ig = gx0 + tx, jg = gy0 + ty;
    if (!active || ig >= w || jg >= h) return;
    const float du = T.du[ty + 1][tx + 1], dv = T.dv[ty + 1][tx + 1];
    const float Iz = P.wIz.at(jg, ig), Ix = P.wIx.at(jg, ig), Ixz = P.wIxz.at(jg, ig), Ixy = P.wIxy.at(jg, ig);
    const float Ixx = P.wIxx.at(jg, ig), Iy = P.wIy.at(jg, ig), Iyz = P.wIyz.at(jg, ig), Iyy = P.wIyy.at(jg, ig);
    const float q0 = __fmaf_rn(dv, Iy, __fmaf_rn(du, Ix, Iz));
    const float q1 = __fmaf_rn(dv, Ixy, __fmaf_rn(du, Ixx, Ixz));
    const float q2 = __fmaf_rn(dv, Iyy, __fmaf_rn(du, Ixy, Iyz));
    const float r2 = __fadd_rn(__fmaf_rn(q0, q0, __fmul_rn(gamma, __fmaf_rn(q1, q1, __fmul_rn(q2, q2)))), EPS2);
    float data_term = __fmul_rn(0.5f, EXACT_RSQ ? __frsqrt_rn(r2) : rsqrtf(r2));
    data_term = __fdiv_rn(data_term, alpha);

    const float sx = S.sx[ty][tx], sxr = S.sx[ty][tx + 1];
    const float sy = S.sy[ty][tx], syu = S.sy[ty + 1][tx];

    // which product of a sum of two products is fused is nvcc's choice, pinned here term by term
    P.num_dudv.at(jg, ig) = __fmul_rn(data_term, __fmaf_rn(Ix, Iy, __fmul_rn(__fmul_rn(gamma, Ixy), __fadd_rn(Ixx, Iyy))));
    P.num_u.at(jg, ig) = __fmul_rn(data_term, __fmaf_rn(Ix, Iz, __fmul_rn(gamma, __fmaf_rn(Ixx, Ixz, __fmul_rn(Ixy, Iyz)))));
    P.num_v.at(jg, ig) = __fmul_rn(data_term, __fmaf_rn(Iy, Iz, __fmul_rn(gamma, __fmaf_rn(Ixy, Ixz, __fmul_rn(Iyy, Iyz)))));
    // data_term * den + dsum is one rounding
    const float den_u = __fmaf_rn(Ix, Ix, __fmul_rn(gamma, __fmaf_rn(Ixy, Ixy, __fmul_rn(Ixx, Ixx))));
    const float den_v = __fmaf_rn(Iy, Iy, __fmul_rn(gamma, __fmaf_rn(Ixy, Ixy, __fmul_rn(Iyy, Iyy))));
    P.sx.at(jg, ig) = sx;
    P.sy.at(jg, ig) = sy;
    const float dsum = __fadd_rn(__fadd_rn(__fadd_rn(sx, sxr), sy), syu);
    P.inv_u.at(jg, ig) = __frcp_rn(__fmaf_rn(data_term, den_u, dsum));
    P.inv_v.at(jg, ig) = __frcp_rn(__fmaf_rn(data_term, den_v, dsum));
}

template <bool EXACT_RSQ>
__global__ void __launch_bounds__(PB_X *PB_Y) k_brox_prepare(BroxLevelPlanes P, int h, int w, float alpha, float gamma) {
    __shared__ PrepShared S;
    brox_prepare_chunk<false, EXACT_RSQ>(P, h, w, alpha, gamma, blockIdx.x * PB_X, blockIdx.y * PB_Y, threadIdx.y * PB_X + threadIdx.x, S,
                              true);
}

// ---------------------------------------------------------------------------------------------
// One SOR cell update (NB:501-547) with every rounding made explicit, shared by the three solver kernels
// so that they agree bit for bit.  U* / V* are the neighbours' (u + du) / (v + dv); usum = u * ssum and
// w_u = omega * inv_denom_u are per-cell constants of an inner step (the products the reference's
// left-to-right expression forms first), so the register-resident kernel can hoist them.
// ---------------------------------------------------------------------------------------------
struct SorConst {
    float s_l, s_r, s_u, s_d;   // diffusivities towards the four neighbours (0 beyond the image)
    float usum, vsum;           // u * (s_l + s_r + s_u + s_d), v * (...)
    float num_u, num_v, num_dudv;
    float w_u, w_v;             // omega * inv_denom
};
__device__ __forceinline__ float brox_ssum(float s_l, float s_r, float s_u, float s_d) {
    return __fadd_rn(__fadd_rn(__fadd_rn(s_l, s_r), s_u), s_d);
}
__device__ __forceinline__ void brox_sor_cell(const SorConst &c, float Ul, float Uu, float Ur, float Ud, float Vl,
                                              float Vu, float Vr, float Vd, float one_minus_omega, float &du,
                                              float &dv) {
    float t = __fmul_rn(c.s_l, Ul);
    t = __fmaf_rn(c.s_u, Uu, t);
    t = __fmaf_rn(c.s_r, Ur, t);
    t = __fmaf_rn(c.s_d, Ud, t);
    t = __fsub_rn(t, c.usum);
    t = __fsub_rn(t, c.num_u);
    t = __fmaf_rn(-c.num_dudv, dv, t);
    du = __fmaf_rn(c.w_u, t, __fmul_rn(one_minus_omega, du));
    t = __fmul_rn(c.s_l, Vl);
    t = __fmaf_rn(c.s_u, Vu, t);
    t = __fmaf_rn(c.s_r, Vr, t);
    t = __fmaf_rn(c.s_d, Vd, t);
    t = __fsub_rn(t, c.vsum);
    t = __fsub_rn(t, c.num_v);
    t = __fmaf_rn(-c.num_dudv, du, t);  // uses the NEW du (NB:538-545)
    dv = __fmaf_rn(c.w_v, t, __fmul_rn(one_minus_omega, dv));
}

// ---------------------------------------------------------------------------------------------
// one red or black half sweep (NB:479-554), omega = 1.99
// ---------------------------------------------------------------------------------------------
template <int IS_BLACK>
__global__ void __launch_bounds__(256) k_brox_sor(BroxLevelPlanes P, Plane du_in, Plane dv_in, Plane du_out,
                                                  Plane dv_out, int h, int w, float omega) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    float du = du_in.at(j, i), dv = dv_in.at(j, i);
    if (((i + j) & 1) == IS_BLACK) {
        const int ir = i < w - 1 ? i + 1 : i, il = i > 0 ? i - 1 : i;
        const int ju = j < h - 1 ? j + 1 : j, jd = j > 0 ? j - 1 : j;
        SorConst c;
        c.s_l = P.sx.at(j, i);
        c.s_d = P.sy.at(j, i);
        c.s_r = i < w - 1 ? P.sx.at(j, ir) : 0.0f;
        c.s_u = j < h - 1 ? P.sy.at(ju, i) : 0.0f;
        const float ssum = brox_ssum(c.s_l, c.s_r, c.s_u, c.s_d);
        c.usum = __fmul_rn(P.u.at(j, i), ssum);
        c.vsum = __fmul_rn(P.v.at(j, i), ssum);
        c.num_u = P.num_u.at(j, i);
        c.num_v = P.num_v.at(j, i);
        c.num_dudv = P.num_dudv.at(j, i);
        c.w_u = __fmul_rn(omega, P.inv_u.at(j, i));
        c.w_v = __fmul_rn(omega, P.inv_v.at(j, i));
        auto U = [&](int y, int x) { return __fadd_rn(P.u.at(y, x), du_in.at(y, x)); };
        auto V = [&](int y, int x) { return __fadd_rn(P.v.at(y, x), dv_in.at(y, x)); };
        brox_sor_cell(c, U(j, il), U(ju, i), U(j, ir), U(jd, i), V(j, il), V(ju, i), V(j, ir), V(jd, i), 1.0f - omega, du,
                      dv);
    }
    du_out.at(j, i) = du;
    dv_out.at(j, i) = dv;
}

// ---------------------------------------------------------------------------------------------
// Fused red-black SOR: `iters` full iterations (2*iters half sweeps) per launch on a 64x64 region held in
// shared memory.  Each half sweep consumes one halo cell per side, so the centre (64 - 4*iters)^2 tile
// is exact (bit-identical to `iters` pairs of k_brox_sor launches: a colour's update reads only the
// other colour, so updating in place equals the reference's ping-pong).  A level that fits in one region
// needs no halo at all and runs all solver iterations of an inner step in one launch.
// ---------------------------------------------------------------------------------------------
constexpr int SR = 64;           // region edge
constexpr int S_THREADS = 512;

__global__ void __launch_bounds__(S_THREADS, 1)
    k_brox_sor_fused_pp(BroxLevelPlanes P, Plane du_out, Plane dv_out, int h, int w, float omega, int iters, int halo,
                        int tile) {
    extern __shared__ float ssm[];
    float *s_du = ssm, *s_dv = ssm + SR * SR, *s_u = ssm + 2 * SR * SR, *s_v = ssm + 3 * SR * SR;
    float *s_sx = ssm + 4 * SR * SR, *s_sy = ssm + 5 * SR * SR, *s_iu = ssm + 6 * SR * SR, *s_iv = ssm + 7 * SR * SR;
    float *s_nu = ssm + 8 * SR * SR, *s_nv = ssm + 9 * SR * SR, *s_nd = ssm + 10 * SR * SR;
    const int tid = threadIdx.x;
    const int gx0 = blockIdx.x * tile - halo, gy0 = blockIdx.y * tile - halo;

    for (int idx = tid; idx < SR * SR; idx += S_THREADS) {
        const int ry = idx >> 6, rx = idx & 63;
        const int gy = gy0 + ry, gx = gx0 + rx;
        const bool in = gx >= 0 && gy >= 0 && gx < w && gy < h;
        s_du[idx] = in ? P.du.at(gy, gx) : 0.f;
        s_dv[idx] = in ? P.dv.at(gy, gx) : 0.f;
        s_u[idx] = in ? P.u.at(gy, gx) : 0.f;
        s_v[idx] = in ? P.v.at(gy, gx) : 0.f;
        s_sx[idx] = in ? P.sx.at(gy, gx) : 0.f;
        s_sy[idx] = in ? P.sy.at(gy, gx) : 0.f;
        s_iu[idx] = in ? P.inv_u.at(gy, gx) : 0.f;
        s_iv[idx] = in ? P.inv_v.at(gy, gx) : 0.f;
        s_nu[idx] = in ? P.num_u.at(gy, gx) : 0.f;
        s_nv[idx] = in ? P.num_v.at(gy, gx) : 0.f;
        s_nd[idx] = in ? P.num_dudv.at(gy, gx) : 0.f;
    }
    __syncthreads();

    for (int sweep = 0; sweep < 2 * iters; ++sweep) {
        const int colour = sweep & 1;  // sor_pass<0> first, then sor_pass<1> (NB:915-922)
        for (int c = tid; c < SR * SR / 2; c += S_THREADS) {
            const int ry = c >> 5;
            const int rx = ((c & 31) << 1) + ((ry + gy0 + gx0 + colour) & 1);  // (gx + gy) % 2 == colour
            const int gy = gy0 + ry, gx = gx0 + rx;
            if (gx < 0 || gy < 0 || gx >= w || gy >= h) continue;
            // region-edge cells read clamped region neighbours: their values are stale, but they lie in the halo
            const int idx = ry * SR + rx;
            const int il = (gx > 0 && rx > 0) ? idx - 1 : idx, ir = (gx < w - 1 && rx < SR - 1) ? idx + 1 : idx;
            const int id = (gy > 0 && ry > 0) ? idx - SR : idx, iu = (gy < h - 1 && ry < SR - 1) ? idx + SR : idx;
            SorConst cc;
            cc.s_l = s_sx[idx];
            cc.s_d = s_sy[idx];
            cc.s_r = gx < w - 1 ? s_sx[ir] : 0.0f;
            cc.s_u = gy < h - 1 ? s_sy[iu] : 0.0f;
            const float ssum = brox_ssum(cc.s_l, cc.s_r, cc.s_u, cc.s_d);
            cc.usum = __fmul_rn(s_u[idx], ssum);
            cc.vsum = __fmul_rn(s_v[idx], ssum);
            cc.num_u = s_nu[idx];
            cc.num_v = s_nv[idx];
            cc.num_dudv = s_nd[idx];
            cc.w_u = __fmul_rn(omega, s_iu[idx]);
            cc.w_v = __fmul_rn(omega, s_iv[idx]);
            float du = s_du[idx], dv = s_dv[idx];
            auto U = [&](int q) { return __fadd_rn(s_u[q], s_du[q]); };
            auto V = [&](int q) { return __fadd_rn(s_v[q], s_dv[q]); };
            brox_sor_cell(cc, U(il), U(iu), U(ir), U(id), V(il), V(iu), V(ir), V(id), 1.0f - omega, du, dv);
            s_du[idx] = du;
            s_dv[idx] = dv;
        }
        __syncthreads();
    }

    for (int idx = tid; idx < tile * tile; idx += S_THREADS) {
        const int ty = idx / tile, tx = idx - ty * tile;
        const int gy = gy0 + halo + ty, gx = gx0 + halo + tx;
        if (gx < w && gy < h) {
            du_out.at(gy, gx) = s_du[(halo + ty) * SR + halo + tx];
            dv_out.at(gy, gx) = s_dv[(halo + ty) * SR + halo + tx];
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Register-resident fused SOR (default path).  Same region / halo scheme as k_brox_sor_fused_pp, but a
// thread owns a 2-column x 4-row patch of the 64x64 region and keeps its eight cells' (du, dv, u + du,
// v + dv) and hoisted constants in registers; the rest of the per-cell constants sit in shared memory in
// a colour-major layout that every warp reads conflict-free with 128-bit loads.  Horizontal neighbours
// come from the own patch or one warp shuffle, vertical neighbours from the own patch except across the
// 4-row boundary, where the two boundary rows are exchanged through shared memory (one barrier per half
// sweep).  Shared-memory traffic per cell update drops from 31 two-way-conflicting word loads to two
// conflict-free 128-bit loads.  Bit-identical to the other two solver kernels (brox_sor_cell).
// ---------------------------------------------------------------------------------------------
struct SorRegs {
    float du, dv, U, V, u, v, usum, vsum, w_v;
};

// No border logic is needed inside the sweep: wherever the reference clamps a neighbour index (image border) the
// matching diffusivity is zero (sx = 0 at i = 0, sy = 0 at j = 0 by construction; s_right / s_up are zeroed
// at the far edges on load), so the clamped neighbour contributes exactly +-0 whatever finite value is read;
// cells outside the image carry all-zero constants and therefore stay at du = dv = 0.
template <int CP0>
__device__ __forceinline__ void brox_half_sweep(SorRegs (&c)[4][2], const float4 *__restrict__ sS,
                                                const float4 *__restrict__ sN, float *__restrict__ xU,
                                                float *__restrict__ xV, int lane, int ry0, int rx0,
                                                float one_minus_omega) {
    // neighbours across the 4-row boundary (the other colour: written in the previous half sweep)
    constexpr int cpT = CP0, cpB = CP0 ^ 1;  // active column in patch rows 0 and 3
    const int below = (ry0 > 0 ? ry0 - 1 : ry0) * SR + rx0 + cpT;
    const int above = (ry0 + 4 < SR ? ry0 + 4 : ry0 + 3) * SR + rx0 + cpB;
    const float Ud0 = xU[below], Vd0 = xV[below];
    const float Uu3 = xU[above], Vu3 = xV[above];
    const float4 *pS = sS + (ry0 * 2) * 32 + lane, *pN = sN + (ry0 * 2) * 32 + lane;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        constexpr int dummy = 0;
        (void)dummy;
        const int cp = (CP0 ^ r) & 1;  // compile-time after unrolling
        // horizontal neighbours: the other column of the own patch and the adjacent lane's (a region-edge lane
        // gets its own value back from the shuffle: stale but finite, and it lies in the halo)
        const float Uo = c[r][cp ^ 1].U, Vo = c[r][cp ^ 1].V;
        float Ul, Ur, Vl, Vr;
        if (cp == 0) {
            Ul = __shfl_up_sync(0xffffffffu, Uo, 1);
            Vl = __shfl_up_sync(0xffffffffu, Vo, 1);
            Ur = Uo;
            Vr = Vo;
        } else {
            Ur = __shfl_down_sync(0xffffffffu, Uo, 1);
            Vr = __shfl_down_sync(0xffffffffu, Vo, 1);
            Ul = Uo;
            Vl = Vo;
        }
        const float Ud = r == 0 ? Ud0 : c[r > 0 ? r - 1 : 0][cp].U;
        const float Vd = r == 0 ? Vd0 : c[r > 0 ? r - 1 : 0][cp].V;
        const float Uu = r == 3 ? Uu3 : c[r < 3 ? r + 1 : 3][cp].U;
        const float Vu = r == 3 ? Vu3 : c[r < 3 ? r + 1 : 3][cp].V;
        SorRegs &me = c[r][cp];
        const float4 S = pS[(r * 2 + cp) * 32], N = pN[(r * 2 + cp) * 32];
        SorConst k;
        k.s_l = S.x; k.s_r = S.y; k.s_u = S.z; k.s_d = S.w;
        k.num_u = N.x; k.num_v = N.y; k.num_dudv = N.z; k.w_u = N.w;
        k.usum = me.usum; k.vsum = me.vsum; k.w_v = me.w_v;
        brox_sor_cell(k, Ul, Uu, Ur, Ud, Vl, Vu, Vr, Vd, one_minus_omega, me.du, me.dv);
        me.U = __fadd_rn(me.u, me.du);
        me.V = __fadd_rn(me.v, me.dv);
    }
    // publish the updated boundary cells for the neighbouring warps' next half sweep
    xU[ry0 * SR + rx0 + cpT] = c[0][cpT].U;
    xV[ry0 * SR + rx0 + cpT] = c[0][cpT].V;
    xU[(ry0 + 3) * SR + rx0 + cpB] = c[3][cpB].U;
    xV[(ry0 + 3) * SR + rx0 + cpB] = c[3][cpB].V;
}

// One 64 x 64 region: load, `iters` full iterations in registers, store the centre tile.  (bx, by) = region index.
// CG: operands written by other CTAs of the same launch (du, dv and everything k_brox_prepare produces) are read through L2.
template <bool CG>
__device__ __forceinline__ void brox_sor_region(const BroxLevelPlanes &P, Plane du_out, Plane dv_out, int h, int w, float omega,
                                                int iters, int halo, int tile, int bx, int by, float4 *sor4) {
    float4 *sS = sor4;                 // [row][colour-parity][k] : s_l, s_r, s_u, s_d
    float4 *sN = sor4 + SR * SR;       // same layout            : num_u, num_v, num_dudv, omega * inv_u
    float *xU = reinterpret_cast<float *>(sor4 + 2 * SR * SR);  // boundary-row exchange, [row][col]
    float *xV = xU + SR * SR;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rx0 = 2 * lane, ry0 = 4 * warp;
    const int gx0 = bx * tile - halo, gy0 = by * tile - halo;  // both even

    SorRegs c[4][2];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int gy = gy0 + ry0 + r, gx = gx0 + rx0 + q;
            const bool in = gx >= 0 && gy >= 0 && gx < w && gy < h;
            SorRegs &m = c[r][q];
            float4 S = make_float4(0.f, 0.f, 0.f, 0.f), N = make_float4(0.f, 0.f, 0.f, 0.f);
            m.du = m.dv = m.u = m.v = m.usum = m.vsum = m.w_v = 0.f;
            if (in) {
                m.du = brox_ld<CG>(P.du, gy, gx);
                m.dv = brox_ld<CG>(P.dv, gy, gx);
                m.u = P.u.at(gy, gx);
                m.v = P.v.at(gy, gx);
                S.x = brox_ld<CG>(P.sx, gy, gx);
                S.w = brox_ld<CG>(P.sy, gy, gx);
                S.y = gx < w - 1 ? brox_ld<CG>(P.sx, gy, gx + 1) : 0.0f;
                S.z = gy < h - 1 ? brox_ld<CG>(P.sy, gy + 1, gx) : 0.0f;
                const float ssum = brox_ssum(S.x, S.y, S.z, S.w);
                m.usum = __fmul_rn(m.u, ssum);
                m.vsum = __fmul_rn(m.v, ssum);
                N.x = brox_ld<CG>(P.num_u, gy, gx);
                N.y = brox_ld<CG>(P.num_v, gy, gx);
                N.z = brox_ld<CG>(P.num_dudv, gy, gx);
                N.w = __fmul_rn(omega, brox_ld<CG>(P.inv_u, gy, gx));
                m.w_v = __fmul_rn(omega, brox_ld<CG>(P.inv_v, gy, gx));
            }
            m.U = __fadd_rn(m.u, m.du);
            m.V = __fadd_rn(m.v, m.dv);
            const int slot = ((ry0 + r) * 2 + q) * 32 + lane;
            sS[slot] = S;
            sN[slot] = N;
            if (r == 0 || r == 3) {
                xU[(ry0 + r) * SR + rx0 + q] = m.U;
                xV[(ry0 + r) * SR + rx0 + q] = m.V;
            }
        }
    }
    __syncthreads();

    const float omo = 1.0f - omega;
    // colour 0 first (sor_pass<0>, NB:915-922): cells with (gx + gy) even; gx0 is even, so in patch row 0 the
    // active column is (colour ^ gy0 ^ ry0) & 1 = (colour ^ gy0) & 1 -- uniform over the CTA
    const int par = gy0 & 1;
    // warps whose four rows lie outside the image hold only zero cells: they skip the arithmetic (small levels
    // occupy a corner of the region) but keep the barrier
    const bool live = gy0 + ry0 < h && gy0 + ry0 + 3 >= 0;
    for (int sweep = 0; sweep < 2 * iters; ++sweep) {
        if (live) {
            if (((sweep ^ par) & 1) == 0)
                brox_half_sweep<0>(c, sS, sN, xU, xV, lane, ry0, rx0, omo);
            else
                brox_half_sweep<1>(c, sS, sN, xU, xV, lane, ry0, rx0, omo);
        }
        __syncthreads();
    }

#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int ry = ry0 + r, gy = gy0 + ry;
        if (ry < halo || ry >= halo + tile || gy >= h) continue;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int rx = rx0 + q, gx = gx0 + rx;
            if (rx < halo || rx >= halo + tile || gx >= w) continue;
            du_out.at(gy, gx) = c[r][q].du;
            dv_out.at(gy, gx) = c[r][q].dv;
        }
    }
}

__global__ void __launch_bounds__(S_THREADS, 1)
    k_brox_sor_reg(BroxLevelPlanes P, Plane du_out, Plane dv_out, int h, int w, float omega, int iters, int halo,
                   int tile) {
    extern __shared__ float4 sor4[];
    brox_sor_region<false>(P, du_out, dv_out, h, w, omega, iters, halo, tile, blockIdx.x, blockIdx.y, sor4);
}

// ---------------------------------------------------------------------------------------------
// Cooperative level kernel: ALL inner iterations of a level in one launch -- per inner iteration the prepare pass over
// the level's 32 x 8 chunks (two at a time per CTA), a grid-wide barrier, the register-resident solver on the CTA's
// region (all solver iterations), a grid-wide barrier.  For the levels whose solver takes every iteration in one launch
// (13 of the 19 levels of a 720p pyramid; they are bound by launch floors, not by work) this replaces 2 x inner launches
// and their gaps.  Opt-in (kernel_path 3), see BroxEngine::solve.  Launched with cudaLaunchCooperativeKernel (co-residency is what makes the spin barrier legal); the
// barrier counter is zeroed by a memset node in front of every launch.  Same device functions as the stand-alone kernels:
// bit-identical to them.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void brox_grid_barrier(unsigned *counter, unsigned nblocks, unsigned &epoch) {
    __syncthreads();
    ++epoch;
    if (threadIdx.x == 0) {
        __threadfence();  // this CTA's stores before its arrival
        atomicAdd(counter, 1u);
        const unsigned target = epoch * nblocks;
        unsigned seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
    }
    __syncthreads();
}

template <bool EXACT_RSQ>
__global__ void __launch_bounds__(S_THREADS, 1)
    k_brox_level_coop(BroxLevelPlanes P, Plane dun, Plane dvn, int h, int w, float alpha, float gamma, float omega, int inner,
                      int iters, int halo, int tile, int tiles_x, unsigned *barrier) {
    extern __shared__ float4 sor4[];
    __shared__ PrepShared PS[2];
    const int tid = threadIdx.x, half = tid >> 8, t256 = tid & 255;
    const int chunks_x = (w + PB_X - 1) / PB_X, chunks_y = (h + PB_Y - 1) / PB_Y, nchunks = chunks_x * chunks_y;
    const int by = blockIdx.x / tiles_x, bx = blockIdx.x - by * tiles_x;
    unsigned epoch = 0;
    Plane cdu = P.du, cdv = P.dv, ndu = dun, ndv = dvn;
    for (int in = 0; in < inner; ++in) {
        BroxLevelPlanes Q = P;
        Q.du = cdu;
        Q.dv = cdv;
        for (int c0 = 2 * blockIdx.x; c0 < nchunks; c0 += 2 * gridDim.x) {  // uniform trip count over the CTA
            const int c = c0 + half;
            const bool active = c < nchunks;
            const int cy = active ? c / chunks_x : 0, cx = active ? c - cy * chunks_x : 0;
            brox_prepare_chunk<true, EXACT_RSQ>(Q, h, w, alpha, gamma, cx * PB_X, cy * PB_Y, t256, PS[half], active);
            __syncthreads();  // the tiles are reused by the next round
        }
        brox_grid_barrier(barrier, gridDim.x, epoch);
        brox_sor_region<true>(Q, ndu, ndv, h, w, omega, iters, halo, tile, bx, by, sor4);
        Plane t1 = cdu; cdu = ndu; ndu = t1;
        Plane t2 = cdv; cdv = ndv; ndv = t2;
        brox_grid_barrier(barrier, gridDim.x, epoch);
    }
}

// u += du ; v += dv  (NB:929-931), in place
__global__ void __launch_bounds__(256) k_brox_add(Plane u, Plane v, Plane du, Plane dv, int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    u.at(y, x) = __fadd_rn(u.at(y, x), du.at(y, x));
    v.at(y, x) = __fadd_rn(v.at(y, x), dv.at(y, x));
}

// bicubic prolongation (NS:2172-2231) fused with ScaleVector (NB:952-961); u and v per launch
__device__ __forceinline__ float brox_bicubic_coeff(float x_) {
    const float x = fabsf(x_);
    if (x <= 1.0f) return __fmaf_rn(__fmul_rn(x, x), __fmaf_rn(x, 1.5f, -2.5f), 1.0f);
    if (x < 2.0f) return __fmaf_rn(x, __fmaf_rn(x, __fmaf_rn(x, -0.5f, 2.5f), -4.0f), 2.0f);
    return 0.0f;
}

__global__ void __launch_bounds__(256) k_brox_prolong(Plane su, Plane sv, int sh, int sw, Plane du, Plane dv, int dh,
                                                      int dw, float scale, float mul) {
    const int ix = blockIdx.x * blockDim.x + threadIdx.x;
    const int iy = blockIdx.y * blockDim.y + threadIdx.y;
    if (ix >= dw || iy >= dh) return;
    const Plane src = blockIdx.z ? sv : su;
    const float rw = (float)sw, rh = (float)sh;
    // x = scale * ix is never rounded on its own: every use fuses the product (x - 2, x + 2, x - cx)
    const float fx = (float)ix, fy = (float)iy;
    const float xmin = fmaxf(ceilf(__fmaf_rn(fx, scale, -2.0f)), 0.0f), xmax = fminf(floorf(__fmaf_rn(fx, scale, 2.0f)), __fsub_rn(rw, 1.0f));
    const float ymin = fmaxf(ceilf(__fmaf_rn(fy, scale, -2.0f)), 0.0f), ymax = fminf(floorf(__fmaf_rn(fy, scale, 2.0f)), __fsub_rn(rh, 1.0f));
    float sum = 0.0f, wsum = 0.0f;
    for (float cy = ymin; cy <= ymax; cy = __fadd_rn(cy, 1.0f)) {
        for (float cx = xmin; cx <= xmax; cx = __fadd_rn(cx, 1.0f)) {
            float wx = brox_bicubic_coeff(__fmaf_rn(fx, scale, -cx));
            const float wy = brox_bicubic_coeff(__fmaf_rn(fy, scale, -cy));
            wx = __fmul_rn(wx, wy);
            sum = __fmaf_rn(wx, __ldg(&src.at((int)cy, (int)cx)), sum);
            wsum = __fadd_rn(wsum, wx);
        }
    }
    const float r = (!wsum) ? 0.f : __fdiv_rn(sum, wsum);
    (blockIdx.z ? dv : du).at(iy, ix) = __fmul_rn(r, mul);
}

// ---------------------------------------------------------------------------------------------
// host engine
// ---------------------------------------------------------------------------------------------
struct BLevel {
    int rows = 0, cols = 0;
    Plane I0, I1;
};

class BroxEngine : public b2f_handle {
public:
    explicit BroxEngine(const b2f_brox_params &p) : P(p) { algo = ALGO_BROX; }
    b2f_brox_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    const char *default_name() const override { return "DenseOpticalFlow.BroxOpticalFlow"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"brox_sor", "brox_prepare", "brox_derivatives", "brox_pyramid"};
        return (cls >= 0 && cls < 4) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        Layout L;
        return layout(rows, cols, true, L);
    }

private:
    struct Layout {
        int rows = 0, cols = 0;
        b2f_brox_params P{};
        std::vector<BLevel> levels;
        float *shared[32] = {};
    };
    Layout L_;
    enum { S_IX = 0, S_IXX, S_IX0, S_IY, S_IYY, S_IY0, S_IXY, S_U, S_V, S_UN, S_VN, S_DU, S_DV, S_DUN, S_DVN, S_SX, S_SY,
           S_INVU, S_INVV, S_NDUDV, S_WIZ, S_WIX, S_WIXZ, S_WIXY, S_WIXX, S_WIY, S_WIYZ, S_WIYY, S_COUNT };
    float *extra_[2] = {};  // num_u, num_v
    unsigned *coop_barrier_ = nullptr;  // arrival counter of the cooperative level kernel (zeroed before every launch)
    int coop_max_blocks_[2] = {-1, -1}; // co-resident CTAs of k_brox_level_coop<aux_path == 1> on this device (0: unsupported)
    bool coop_ok(int blocks, bool exact_rsq);
    int final_ui_ = 0;      // which (u, v) buffer pair holds the result (fixed by the level count)

    struct GraphKey {
        int rows, cols;
        b2f_brox_params P;
        EngineKnobs knobs;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && same_knobs(knobs, o.knobs) && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;

    size_t layout(int rows, int cols, bool counting, Layout &L);
    cudaError_t ensure_workspace(int rows, int cols);
    Plane sp(int idx, int cols) const { return Plane{L_.shared[idx], plane_pitch(cols)}; }
    void solve(Ctx &c);
};

size_t BroxEngine::layout(int rows, int cols, bool counting, Layout &L) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.rows = rows;
    L.cols = cols;
    L.P = P;
    L.levels.clear();
    // pyramid sizes, NB:730-785: ceilf(src * scale) with a cumulative float scale
    const float sf = static_cast<float>(P.scale_factor);
    float scale = 1.0f * sf;
    BLevel l0;
    l0.rows = rows;
    l0.cols = cols;
    l0.I0 = A.plane(rows, cols);
    l0.I1 = A.plane(rows, cols);
    L.levels.push_back(l0);
    int pw = cols, ph = rows;
    while (pw > 15 && ph > 15 && (int)L.levels.size() < P.outer_iterations) {
        BLevel lv;
        lv.cols = static_cast<int>(ceilf(cols * scale));
        lv.rows = static_cast<int>(ceilf(rows * scale));
        lv.I0 = A.plane(lv.rows, lv.cols);
        lv.I1 = A.plane(lv.rows, lv.cols);
        L.levels.push_back(lv);
        scale *= sf;
        pw = lv.cols;
        ph = lv.rows;
    }
    for (int i = 0; i < S_COUNT; ++i) L.shared[i] = A.plane(rows, cols).p;
    float *a = A.plane(rows, cols).p, *b = A.plane(rows, cols).p;
    unsigned *bar = static_cast<unsigned *>(A.bytes(256));
    if (!counting) {
        extra_[0] = a;
        extra_[1] = b;
        coop_barrier_ = bar;
    }
    return A.used();
}

cudaError_t BroxEngine::ensure_workspace(int rows, int cols) {
    if (L_.rows == rows && L_.cols == cols && same_params(L_.P, P) && arena.capacity() > 0)
        return cudaSuccess;
    Layout tmp;
    const size_t need = layout(rows, cols, true, tmp);
    graph_.destroy();
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    layout(rows, cols, false, L_);
    return cudaSuccess;
}

bool BroxEngine::coop_ok(int blocks, bool exact_rsq) {
    int &max_blocks = coop_max_blocks_[exact_rsq];
    if (max_blocks < 0) {
        max_blocks = 0;
        int dev = 0, coop = 0, per_sm = 0;
        const size_t smem = sizeof(float) * 10 * SR * SR;
        auto kern = exact_rsq ? k_brox_level_coop<true> : k_brox_level_coop<false>;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev) == cudaSuccess && coop &&
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess &&
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, S_THREADS, smem) == cudaSuccess)
            max_blocks = per_sm * sm_count();
        cudaGetLastError();
        if (getenv("B2F_BROX_NO_COOP")) max_blocks = 0;
    }
    return blocks > 0 && blocks <= max_blocks;
}

void BroxEngine::solve(Ctx &c) {
    const dim3 block(32, 8);
    const size_t sor_smem = sizeof(float) * 11 * SR * SR;
    const size_t sor_reg_smem = sizeof(float) * 10 * SR * SR;  // two float4 constant arrays + two exchange planes
    const float inv_sf = 1.0f / static_cast<float>(P.scale_factor);  // kernels get 1/xFactor (NS:2264,2270)
    const int nl = static_cast<int>(L_.levels.size());
    // restriction, level by level from the previous one
    for (int l = 1; l < nl; ++l) {
        const BLevel &a = L_.levels[l - 1], &b = L_.levels[l];
        const dim3 grid(div_up(b.cols, 32), div_up(b.rows, 8), 2);
        B2F_LAUNCH(c, CLS_PYR, 2.0 * 4.0 * ((double)a.rows * a.cols + (double)b.rows * b.cols), k_brox_supersample, grid,
                   block, 0, a.I0, a.I1, a.rows, a.cols, b.I0, b.I1, b.rows, b.cols, inv_sf);
    }
    int ui = 0;  // (u, v) live in S_U/S_V (0) or S_UN/S_VN (1)
    {
        const BLevel &lc = L_.levels[nl - 1];
        fill_plane(c, sp(S_U, lc.cols), lc.rows, lc.cols, 0.f);
        fill_plane(c, sp(S_V, lc.cols), lc.rows, lc.cols, 0.f);
    }
    for (int l = nl - 1; l >= 0; --l) {
        const BLevel &lv = L_.levels[l];
        const int h = lv.rows, w = lv.cols;
        const double npx = (double)h * w;
        const dim3 grid(div_up(w, 32), div_up(h, 8));
        BroxLevelPlanes T;
        T.I0 = lv.I0; T.I1 = lv.I1;
        T.Ix = sp(S_IX, w); T.Ixx = sp(S_IXX, w); T.Ix0 = sp(S_IX0, w);
        T.Iy = sp(S_IY, w); T.Iyy = sp(S_IYY, w); T.Iy0 = sp(S_IY0, w); T.Ixy = sp(S_IXY, w);
        T.u = sp(ui ? S_UN : S_U, w); T.v = sp(ui ? S_VN : S_V, w);
        T.du = sp(S_DU, w); T.dv = sp(S_DV, w);
        T.sx = sp(S_SX, w); T.sy = sp(S_SY, w); T.inv_u = sp(S_INVU, w); T.inv_v = sp(S_INVV, w);
        T.num_dudv = sp(S_NDUDV, w);
        T.num_u = Plane{extra_[0], plane_pitch(w)};
        T.num_v = Plane{extra_[1], plane_pitch(w)};
        T.wIz = sp(S_WIZ, w); T.wIx = sp(S_WIX, w); T.wIxz = sp(S_WIXZ, w); T.wIxy = sp(S_WIXY, w);
        T.wIxx = sp(S_WIXX, w); T.wIy = sp(S_WIY, w); T.wIyz = sp(S_WIYZ, w); T.wIyy = sp(S_WIYY, w);
        Plane dun = sp(S_DUN, w), dvn = sp(S_DVN, w);

        fill_plane(c, T.du, h, w, 0.f);
        fill_plane(c, T.dv, h, w, 0.f);
        B2F_LAUNCH(c, CLS_DERIV, 24.0 * npx, k_brox_deriv1, grid, block, 0, T.I0, T.I1, T.Ix0, T.Iy0, T.Ix, T.Iy, h, w);
        B2F_LAUNCH(c, CLS_DERIV, 20.0 * npx, k_brox_deriv2, grid, block, 0, T.Ix, T.Iy, T.Ixx, T.Iyy, T.Ixy, h, w);
        B2F_LAUNCH(c, CLS_PREP, 76.0 * npx, k_brox_warp_terms, grid, block, 0, T, h, w);
        const float omega = 1.99f;  // NB:914
        // fused path: up to 12 full iterations per launch (all of them when the level fits one region).
        // A CTA reads its halo from global memory that neighbouring CTAs overwrite with their centre
        // tiles at the end, so launches ping-pong between (du, dv) and (dun, dvn).
        const bool single = w <= SR && h <= SR;  // whole level in one region: no halo, one launch
        // iterations fused per launch: more iterations = fewer launches but a wider halo (smaller tile,
        // more CTAs).  Small and mid levels are latency-bound (one wave), so they take all iterations in
        // one launch; large levels keep the tile big.  Cost model in microseconds: fill ~3, half sweep
        // ~0.35, launch gap ~2, per wave of one CTA per SM.
        int it_best = 5;
        if (!single && knobs.fused_iters > 0) {
            it_best = knobs.fused_iters;
        } else if (!single) {
            double best = 1e30;
            for (int cand = 1; cand <= 12 && cand <= P.solver_iterations; ++cand) {
                const int t = SR - 4 * cand;
                if (t < 8) break;
                const int launches = div_up(P.solver_iterations, cand);
                const double waves = std::ceil((double)div_up(w, t) * div_up(h, t) / (double)sm_count());
                const double cost = launches * (waves * (3.0 + 0.7 * cand) + 2.0);
                if (cost < best) {
                    best = cost;
                    it_best = cand;
                }
            }
        }
        if (it_best > 13) it_best = 13;

        // kernel_path 3 (opt-in): whole level in ONE cooperative launch when every solver iteration of an inner step fits
        // one launch and all its regions are co-resident.  At 720p (10, 77, 10) that is 337 instead of 584 launches per pair,
        // bit-identical, but two software grid barriers per inner step (fence + atomic + acquire polling) and the cooperative
        // launches cost more than the gap a graph leaves between two kernel nodes, and the prepare pass runs on the solver's
        // CTAs only.  The default stays launch-per-step.
        const int it1 = single ? P.solver_iterations : std::min(P.solver_iterations, it_best);
        const int halo1 = single ? 0 : 2 * it1, tile1 = single ? SR : SR - 2 * halo1;
        const int tx1 = single ? 1 : div_up(w, tile1), ty1 = single ? 1 : div_up(h, tile1);
        const bool exact_rsq = knobs.aux_path == 1;
        const bool use_coop = knobs.kernel_path == 3 && it1 == P.solver_iterations && P.solver_iterations > 0 &&
                              P.inner_iterations > 0 && coop_ok(tx1 * ty1, exact_rsq);
        {
            int path = B2F_BROX_PATH_REG, per_launch = single ? P.solver_iterations : std::min(P.solver_iterations, it_best);
            if (use_coop) {
                path = B2F_BROX_PATH_COOP;
            } else if (knobs.kernel_path == 1) {
                path = B2F_BROX_PATH_HALF_SWEEP;
                per_launch = 0;  // a launch is half an iteration
            } else if (knobs.kernel_path == 2) {
                path = B2F_BROX_PATH_SMEM;
            }
            active_paths[l] = path | std::min(per_launch, 255) << 8;
        }
        if (use_coop) {
            c.check(cudaMemsetAsync(coop_barrier_, 0, sizeof(unsigned), c.stream));
            if (c.ok()) {
                c.pre(CLS_SOR, (52.0 * it1 + 104.0) * npx * P.inner_iterations);
                BroxLevelPlanes Q = T;
                float alpha_f = static_cast<float>(P.alpha), gamma_f = static_cast<float>(P.gamma), omega_f = omega;
                int h_ = h, w_ = w, inner_ = P.inner_iterations, iters_ = it1, halo_ = halo1, tile_ = tile1, tx_ = tx1;
                unsigned *bar_ = coop_barrier_;
                void *args[] = {&Q, &dun, &dvn, &h_, &w_, &alpha_f, &gamma_f, &omega_f, &inner_, &iters_, &halo_, &tile_,
                                &tx_, &bar_};
                auto kern = exact_rsq ? k_brox_level_coop<true> : k_brox_level_coop<false>;
                c.check(cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(kern), dim3(tx1 * ty1),
                                                    dim3(S_THREADS), args, sor_reg_smem, c.stream));
                c.post(CLS_SOR);
                c.stats->iterations_run += it1 * P.inner_iterations;
            }
            if (P.inner_iterations & 1) {  // odd number of solver passes: the result sits in the spare pair
                Plane t1 = T.du; T.du = dun; dun = t1;
                Plane t2 = T.dv; T.dv = dvn; dvn = t2;
            }
        }
        for (int in = 0; in < P.inner_iterations && !use_coop; ++in) {
            if (exact_rsq)
                B2F_LAUNCH(c, CLS_PREP, 104.0 * npx, k_brox_prepare<true>, grid, block, 0, T, h, w, static_cast<float>(P.alpha),
                           static_cast<float>(P.gamma));
            else
                B2F_LAUNCH(c, CLS_PREP, 104.0 * npx, k_brox_prepare<false>, grid, block, 0, T, h, w,
                           static_cast<float>(P.alpha), static_cast<float>(P.gamma));
            if (knobs.kernel_path != 1) {
                int left = P.solver_iterations;
                Plane cdu = T.du, cdv = T.dv, ndu = dun, ndv = dvn;
                while (left > 0) {
                    const int it = single ? left : (left < it_best ? left : it_best);
                    const int halo = single ? 0 : 2 * it;
                    const int tile = single ? SR : SR - 2 * halo;
                    const dim3 gs(single ? 1 : div_up(w, tile), single ? 1 : div_up(h, tile));
                    BroxLevelPlanes Q = T;
                    Q.du = cdu;
                    Q.dv = cdv;
                    if (knobs.kernel_path == 2)
                        B2F_LAUNCH(c, CLS_SOR, 52.0 * npx * it, k_brox_sor_fused_pp, gs, dim3(S_THREADS), sor_smem, Q, ndu,
                                   ndv, h, w, omega, it, halo, tile);
                    else
                        B2F_LAUNCH(c, CLS_SOR, 52.0 * npx * it, k_brox_sor_reg, gs, dim3(S_THREADS), sor_reg_smem, Q, ndu,
                                   ndv, h, w, omega, it, halo, tile);
                    Plane t1 = cdu; cdu = ndu; ndu = t1;
                    Plane t2 = cdv; cdv = ndv; ndv = t2;
                    left -= it;
                    c.stats->iterations_run += it;
                }
                if (cdu.p != T.du.p) {  // odd number of launches: result sits in the spare pair -> swap roles
                    Plane t1 = T.du; T.du = dun; dun = t1;
                    Plane t2 = T.dv; T.dv = dvn; dvn = t2;
                }
            } else {
                for (int s = 0; s < P.solver_iterations; ++s) {
                    B2F_LAUNCH(c, CLS_SOR, 26.0 * npx, k_brox_sor<0>, grid, block, 0, T, T.du, T.dv, dun, dvn, h, w, omega);
                    B2F_LAUNCH(c, CLS_SOR, 26.0 * npx, k_brox_sor<1>, grid, block, 0, T, dun, dvn, T.du, T.dv, h, w, omega);
                    c.stats->iterations_run++;
                }
            }
        }
        B2F_LAUNCH(c, CLS_PYR, 24.0 * npx, k_brox_add, grid, block, 0, T.u, T.v, T.du, T.dv, h, w);
        if (l > 0) {
            const BLevel &nx = L_.levels[l - 1];
            Plane nu = sp(ui ? S_U : S_UN, nx.cols), nv = sp(ui ? S_V : S_VN, nx.cols);
            const dim3 g2(div_up(nx.cols, 32), div_up(nx.rows, 8), 2);
            // nppiStResize(..., 1/scale_factor, bicubic) -> kernel scale = scale_factor; then ScaleVector(1/scale_factor)
            B2F_LAUNCH(c, CLS_PYR, 2.0 * 4.0 * (npx + (double)nx.rows * nx.cols), k_brox_prolong, g2, block, 0, T.u, T.v, h,
                       w, nu, nv, nx.rows, nx.cols, 1.0f / inv_sf, inv_sf);
            ui ^= 1;
        }
    }
    final_ui_ = ui;
}

int BroxEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    // preconditions: brox.cpp:134-135 (CV_32FC1, equal size/type), NB:606-617
    if (I0->type != B2F_32FC1 || I1->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    if (!(P.alpha > 0.0) || P.gamma < 0.0 || P.inner_iterations <= 0 || P.outer_iterations <= 0 ||
        P.solver_iterations <= 0)
        return B2F_BAD_ARG;
    if (!(P.scale_factor > 0.0 && P.scale_factor < 1.0)) return B2F_BAD_ARG;
    if (I0->step < (size_t)I0->cols * 4 || I1->step < (size_t)I1->cols * 4 || !flow_step_ok(flow))
        return B2F_BAD_ARG;
    const int rows = I0->rows, cols = I0->cols;
    Ctx c = make_ctx(s);
    static DeviceOnce attrs;
    attrs.run(c, [&] {
        c.check(cudaFuncSetAttribute(k_brox_sor_fused_pp, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(sizeof(float) * 11 * SR * SR)));
        c.check(cudaFuncSetAttribute(k_brox_sor_reg, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(sizeof(float) * 10 * SR * SR)));
    });
    c.check(ensure_workspace(rows, cols));
    if (!c.ok()) return finish(c, s);
    stats.levels = static_cast<int>(L_.levels.size());
    stats.iterations_run = 0;
    active_paths.assign(L_.levels.size(), 0.0);

    const ImageView v0{I0->data, I0->step, rows, cols, I0->type};
    const ImageView v1{I1->data, I1->step, rows, cols, I1->type};
    const ImageView vf = flow_view(flow, rows, cols);
    convert_pair(c, CLS_PYR, v0, v1, L_.levels[0].I0, L_.levels[0].I1, 1.0f);  // NB:714-718 copy into aligned planes

    const bool want_graph = knobs.use_graph && !profiling && s != nullptr;
    if (want_graph) {
        graph_.run(*this, c, s, GraphKey{rows, cols, P, knobs, L_.levels[0].I0.p}, [&](Ctx &g) { solve(g); });
    } else {
        solve(c);
    }
    merge_flow(c, CLS_PYR, sp(final_ui_ ? S_UN : S_U, cols), sp(final_ui_ ? S_VN : S_V, cols), vf);  // brox.cpp:186-187
    return finish(c, s);
}

int BroxEngine::set_param(int id, double v) {
    switch (id) {
        case B2F_BROX_ALPHA: P.alpha = v; break;
        case B2F_BROX_GAMMA: P.gamma = v; break;
        case B2F_BROX_SCALE_FACTOR: P.scale_factor = v; break;
        case B2F_BROX_INNER_ITERATIONS: P.inner_iterations = static_cast<int>(v); break;
        case B2F_BROX_OUTER_ITERATIONS: P.outer_iterations = static_cast<int>(v); break;
        case B2F_BROX_SOLVER_ITERATIONS: P.solver_iterations = static_cast<int>(v); break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

int BroxEngine::get_param(int id, double *v) const {
    switch (id) {
        case B2F_BROX_ALPHA: *v = P.alpha; break;
        case B2F_BROX_GAMMA: *v = P.gamma; break;
        case B2F_BROX_SCALE_FACTOR: *v = P.scale_factor; break;
        case B2F_BROX_INNER_ITERATIONS: *v = P.inner_iterations; break;
        case B2F_BROX_OUTER_ITERATIONS: *v = P.outer_iterations; break;
        case B2F_BROX_SOLVER_ITERATIONS: *v = P.solver_iterations; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

}  // namespace

}  // namespace b2f

extern "C" {

void b2f_brox_default_params(b2f_brox_params *p) {
    if (!p) return;
    p->alpha = 0.197;
    p->gamma = 50.0;
    p->scale_factor = 0.8;
    p->inner_iterations = 5;
    p->outer_iterations = 150;
    p->solver_iterations = 10;
}

int b2f_brox_create(const b2f_brox_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_brox_params d;
    b2f_brox_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::BroxEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
