// tvl1.cu -- cv::cuda::OpticalFlowDual_TVL1 re-implemented for sm_90a.
//
// Reference being replaced (paths relative to opencv_contrib/modules/cudaoptflow):
//   host  src/tvl1flow.cpp:170-382   (calc / calcImpl / procOneScale)
//   dev   src/cuda/tvl1flow.cu:59-348 (centeredGradient, warpBackward, estimateU, estimateDualVariables)
// plus cv::cuda::resize / multiply / merge / calcSum from cudawarping / cudaarithm.
//
// Kernel classes (b2f_stats.class_*):
//   0 iter     inner primal-dual iteration(s)            64 B / px / iteration algorithmic
//   1 warp     centred gradient + bicubic warp + rho/grad 32 B / px / warp
//   2 pyramid  convert + bilinear pyramid                 ~8 B / dst px
//   3 prolong  flow up-sampling (+rescale), split/merge
//   4 reduce   deterministic error reduction (epsilon > 0 only)
#include "common.cuh"
#include "tvl1_math.cuh"
#include "tvl1_blocked.cuh"

#include <cuda.h>  // CUtensorMap (type only; encoded through tma_encode_2d_f32)

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>

namespace b2f {

namespace {

enum { CLS_ITER = 0, CLS_WARP = 1, CLS_PYR = 2, CLS_PROLONG = 3, CLS_REDUCE = 4 };

struct Tvl1Planes {
    Plane I1wx, I1wy, grad, rho_c;
    Plane u1, u2, u3;
    Plane p11, p12, p21, p22, p31, p32;
};

// ---------------------------------------------------------------------------------------------
// warp: fuses centeredGradientKernel + warpBackwardKernel (tvl1flow.cu:59-164).
// The gradients of I1 are formed on the fly from a 6x6 window of I1 (same 0.5f*(a-b) arithmetic
// as the reference's separate gradient pass, so I1x/I1y never touch HBM); taps use clamp
// addressing exactly like the reference's point/clamp textures; I1w is not stored (dead).
// The `grad` plane receives the thresholding constant tvl1_inv_grad(|grad I1w|^2) = 1/|grad|^2 (or the huge stand-in
// for a zero gradient) instead of |grad|^2 itself: every consumer wants the reciprocal, it is constant over a warp's
// inner iterations, and the iteration kernels used to recompute it for every tile of every pass.
// ---------------------------------------------------------------------------------------------
// Border pixels of the warp (window touches the image edge): clamp every tap, then take the clamped-neighbour gradient
// at the clamped tap (point / clamp texture semantics of tvl1flow.cu:106-164).  A real call on purpose.
__device__ __noinline__ void warp_border_taps(const Plane I1, int rows, int cols, int ix, int iy, const float (&kx)[4],
                                              const float (&ky)[4], float &sum, float &sumx, float &sumy) {
    sum = 0.f; sumx = 0.f; sumy = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int cy = clampi(iy + j, 0, rows - 1);
        const int cyp = min(cy + 1, rows - 1), cym = max(cy - 1, 0);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int cx = clampi(ix + i, 0, cols - 1);
            const int cxp = min(cx + 1, cols - 1), cxm = max(cx - 1, 0);
            const float w = kx[i] * ky[j];
            const float v = __ldg(&I1.at(cy, cx));
            const float gx = 0.5f * (__ldg(&I1.at(cy, cxp)) - __ldg(&I1.at(cy, cxm)));
            const float gy = 0.5f * (__ldg(&I1.at(cyp, cx)) - __ldg(&I1.at(cym, cx)));
            sum = __fmaf_rn(w, v, sum);
            sumx = __fmaf_rn(w, gx, sumx);
            sumy = __fmaf_rn(w, gy, sumy);
        }
    }
}

// Keys a = -0.5 weights of the four taps at distances (1 + t, t, 1 - t, 2 - t), t in [0, 1): the reference's bicubic
// polynomials (tvl1flow.cu:89-104) expanded in t (same values up to rounding; t itself is exact, the reference rounds
// t + 1 and 2 - t).
__device__ __forceinline__ void keys_weights(float t, float (&k)[4]) {
    k[0] = ((-0.5f * t + 1.0f) * t - 0.5f) * t;
    k[1] = (1.5f * t - 2.5f) * t * t + 1.0f;
    k[2] = ((-1.5f * t + 2.0f) * t + 0.5f) * t;
    k[3] = (0.5f * t - 0.5f) * t * t;
}

// Separable form of the warp (round 2; aux_path 3, and the fallback for levels smaller than one staged box):
// w_ij = kx[i] * ky[j], so the three weighted sums are row sums r[j] = sum_i kx[i] W[j][i+1] (6 rows),
// rx[j] = sum_i kx[i] (W[j][i+2] - W[j][i]) (4 rows) combined with ky:
//   I1w = sum_j ky[j] r[j+1],  I1wx = 0.5 sum_j ky[j] rx[j+1],  I1wy = 0.5 sum_j ky[j] (r[j+2] - r[j]),
// about half the arithmetic of the tap-by-tap form (the few pixels whose window touches the image border take the
// tap-by-tap loop through an out-of-line call).  Results differ from the tap-by-tap accumulation by rounding only.
// The warp kernel is bound by dependent memory round trips (flow -> window -> stores), not by arithmetic; what the
// separable form buys is registers -- row by row it never holds the 6x6 window, fits 40 registers and runs 6 blocks
// per SM instead of 4.
template <int MINB>
__global__ void __launch_bounds__(256, MINB) k_tvl1_warp_sep(Plane I0, Plane I1, Plane u1p, Plane u2p, Plane I1wx, Plane I1wy,
                                                       Plane grad, Plane rho, int rows, int cols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;

    // all three streaming operands first: the I0 load used to sit behind the first three stores (possible aliasing
    // kept the compiler from hoisting it), a third dependent memory round trip per thread
    const float u1 = __ldg(&u1p.at(y, x));
    const float u2 = __ldg(&u2p.at(y, x));
    const float I0v = __ldg(&I0.at(y, x));
    const float wx = x + u1;
    const float wy = y + u2;
    const float fx = floorf(wx), fy = floorf(wy);
    const int ix = static_cast<int>(fminf(fmaxf(fx, -8.f), cols + 8.f)) - 1;
    const int iy = static_cast<int>(fminf(fmaxf(fy, -8.f), rows + 8.f)) - 1;

    float kx[4], ky[4];
    keys_weights(wx - fx, kx);
    keys_weights(wy - fy, ky);
    float sum, sumx, sumy;
    const float wsum = ((kx[0] + kx[1]) + (kx[2] + kx[3])) * ((ky[0] + ky[1]) + (ky[2] + ky[3]));

    if (ix >= 1 && iy >= 1 && ix + 4 <= cols - 1 && iy + 4 <= rows - 1) {
        const float *base = &I1.at(iy - 1, ix - 1);
        float r[6], rx[4];
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const float *row = base + (size_t)j * I1.pitch;
            const float a1 = __ldg(row + 1), a2 = __ldg(row + 2), a3 = __ldg(row + 3), a4 = __ldg(row + 4);
            r[j] = __fmaf_rn(kx[3], a4, __fmaf_rn(kx[2], a3, __fmaf_rn(kx[1], a2, kx[0] * a1)));
            if (j >= 1 && j <= 4) {
                const float a0 = __ldg(row), a5 = __ldg(row + 5);
                rx[j - 1] = __fmaf_rn(kx[3], a5 - a3, __fmaf_rn(kx[2], a4 - a2, __fmaf_rn(kx[1], a3 - a1, kx[0] * (a2 - a0))));
            }
        }
        sum = __fmaf_rn(ky[3], r[4], __fmaf_rn(ky[2], r[3], __fmaf_rn(ky[1], r[2], ky[0] * r[1])));
        sumx = 0.5f * __fmaf_rn(ky[3], rx[3], __fmaf_rn(ky[2], rx[2], __fmaf_rn(ky[1], rx[1], ky[0] * rx[0])));
        sumy = 0.5f * __fmaf_rn(ky[3], r[5] - r[3], __fmaf_rn(ky[2], r[4] - r[2], __fmaf_rn(ky[1], r[3] - r[1], ky[0] * (r[2] - r[0]))));
    } else {
        warp_border_taps(I1, rows, cols, ix, iy, kx, ky, sum, sumx, sumy);  // out of line: keeps the hot path's registers low
    }

    const float coeff = 1.0f / wsum;
    const float I1w = sum * coeff;
    const float Ix = sumx * coeff;
    const float Iy = sumy * coeff;
    I1wx.at(y, x) = Ix;
    I1wy.at(y, x) = Iy;
    grad.at(y, x) = tvl1_inv_grad(__fmaf_rn(Iy, Iy, __fmul_rn(Ix, Ix)));  // the thresholding constant, not |grad|^2
    rho.at(y, x) = __fsub_rn(__fmaf_rn(-Iy, u2, __fmaf_rn(-Ix, u1, I1w)), I0v);
}

// ---------------------------------------------------------------------------------------------
// Tiled warp kernel (round 2, the default, aux_path 0): the separable warp above executes 325 instructions per pixel, most of
// them 64-bit address arithmetic for its 32 global loads plus the spills of its 40-register cap, and waits on two
// dependent global round trips.  Here one CTA owns a 64 x 32 pixel tile and the
// copy engine stages the (64 + 24) x (32 + 24) window of I1 around it in shared memory (one cp.async.bulk.tensor per
// CTA, issued before the flow is even read).  A pixel whose 6 x 6 tap window lies inside the staged box -- any flow
// up to 9 pixels -- gathers its taps with LDS at compile-time offsets from ONE 32-bit base address; the others take
// the global-memory window (same arithmetic, out of line) or, at the image border, the clamped tap loop.  Same
// expressions in the same order as k_tvl1_warp_sep: bit-identical to it (tested).
// ---------------------------------------------------------------------------------------------
constexpr int WT_W = 64, WT_H = 32, WT_M = 12;
constexpr int WB_W = WT_W + 2 * WT_M, WB_H = WT_H + 2 * WT_M;  // 88 x 56 floats = 19 712 bytes
constexpr int WT_THREADS = 256;

__device__ __forceinline__ uint32_t wt_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wt_mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WT_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WT_DONE;\n\t"
        "bra WT_WAIT;\n\t"
        "WT_DONE:\n\t"
        "}" ::"r"(wt_smem_u32(bar)), "r"(parity) : "memory");
}

// The six-row separable accumulation of k_tvl1_warp_sep on a window whose top-left tap is base[0]; STRIDE > 0: shared
// memory rows of STRIDE floats (every offset an immediate), STRIDE == 0: global rows of `pitch` floats.
template <int STRIDE>
__device__ __forceinline__ void warp_sep_window(const float *base, size_t pitch, const float (&kx)[4], const float (&ky)[4],
                                                float &sum, float &sumx, float &sumy) {
    float r[6], rx[4];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const float *row = STRIDE ? base + j * STRIDE : base + (size_t)j * pitch;
        const float a1 = STRIDE ? row[1] : __ldg(row + 1), a2 = STRIDE ? row[2] : __ldg(row + 2);
        const float a3 = STRIDE ? row[3] : __ldg(row + 3), a4 = STRIDE ? row[4] : __ldg(row + 4);
        r[j] = __fmaf_rn(kx[3], a4, __fmaf_rn(kx[2], a3, __fmaf_rn(kx[1], a2, kx[0] * a1)));
        if (j >= 1 && j <= 4) {
            const float a0 = STRIDE ? row[0] : __ldg(row), a5 = STRIDE ? row[5] : __ldg(row + 5);
            rx[j - 1] = __fmaf_rn(kx[3], a5 - a3, __fmaf_rn(kx[2], a4 - a2, __fmaf_rn(kx[1], a3 - a1, kx[0] * (a2 - a0))));
        }
    }
    sum = __fmaf_rn(ky[3], r[4], __fmaf_rn(ky[2], r[3], __fmaf_rn(ky[1], r[2], ky[0] * r[1])));
    sumx = 0.5f * __fmaf_rn(ky[3], rx[3], __fmaf_rn(ky[2], rx[2], __fmaf_rn(ky[1], rx[1], ky[0] * rx[0])));
    sumy = 0.5f * __fmaf_rn(ky[3], r[5] - r[3], __fmaf_rn(ky[2], r[4] - r[2], __fmaf_rn(ky[1], r[3] - r[1], ky[0] * (r[2] - r[0]))));
}

// Pixels whose window left the staged box (flow beyond the margin) or touches the image border.  A real call on purpose;
// weights and results travel in registers (arrays passed by reference would pin them to the stack in the hot path too).
__device__ __noinline__ float3 warp_slow_taps(const Plane I1, int rows, int cols, int ix, int iy, float kx0, float kx1,
                                              float kx2, float kx3, float ky0, float ky1, float ky2, float ky3) {
    const float kx[4] = {kx0, kx1, kx2, kx3}, ky[4] = {ky0, ky1, ky2, ky3};
    float sum, sumx, sumy;
    if (ix >= 1 && iy >= 1 && ix + 4 <= cols - 1 && iy + 4 <= rows - 1)
        warp_sep_window<0>(&I1.at(iy - 1, ix - 1), (size_t)I1.pitch, kx, ky, sum, sumx, sumy);
    else
        warp_border_taps(I1, rows, cols, ix, iy, kx, ky, sum, sumx, sumy);
    return make_float3(sum, sumx, sumy);
}

// Per-pixel set-up and write-back shared by the two phases of the tiled kernel (same expressions as k_tvl1_warp_sep).
__device__ __forceinline__ void warp_px_setup(int x, int y, float u1, float u2, int rows, int cols, int &ix, int &iy,
                                              float (&kx)[4], float (&ky)[4], float &wsum) {
    const float wx = x + u1;
    const float wy = y + u2;
    const float fx = floorf(wx), fy = floorf(wy);
    ix = static_cast<int>(fminf(fmaxf(fx, -8.f), cols + 8.f)) - 1;
    iy = static_cast<int>(fminf(fmaxf(fy, -8.f), rows + 8.f)) - 1;
    keys_weights(wx - fx, kx);
    keys_weights(wy - fy, ky);
    wsum = ((kx[0] + kx[1]) + (kx[2] + kx[3])) * ((ky[0] + ky[1]) + (ky[2] + ky[3]));
}
__device__ __forceinline__ void warp_px_finish(int x, int y, float u1, float u2, float I0v, float sum, float sumx, float sumy,
                                               float wsum, Plane I1wx, Plane I1wy, Plane grad, Plane rho) {
    const float coeff = 1.0f / wsum;
    const float I1w = sum * coeff;
    const float Ix = sumx * coeff;
    const float Iy = sumy * coeff;
    I1wx.at(y, x) = Ix;
    I1wy.at(y, x) = Iy;
    grad.at(y, x) = tvl1_inv_grad(__fmaf_rn(Iy, Iy, __fmul_rn(Ix, Ix)));  // the thresholding constant, not |grad|^2
    rho.at(y, x) = __fsub_rn(__fmaf_rn(-Iy, u2, __fmaf_rn(-Ix, u1, I1w)), I0v);
}

// Phase 1: every thread walks its 8 pixels; a pixel whose window lies in the staged box is finished on the spot, the
// others (image border, flow beyond the margin) are only queued.  Phase 2: the CTA's queue is worked off one pixel per
// thread.  (Handled in place, a warp on the left / right image edge would make 8 slow calls in a row and hold up the
// end of every launch, whatever the image size.)
template <int MINB>
__global__ void __launch_bounds__(WT_THREADS, MINB)
    k_tvl1_warp_tile(const __grid_constant__ CUtensorMap mapI1, Plane I0, Plane I1, Plane u1p, Plane u2p, Plane I1wx,
                     Plane I1wy, Plane grad, Plane rho, int rows, int cols) {
    __shared__ __align__(128) float win[WB_H * WB_W];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int q_count;
    __shared__ unsigned short q_px[WT_W * WT_H];  // queued pixels, (row in tile) * 64 + (column in tile)
    const int tid = threadIdx.x;
    const int bx0 = blockIdx.x * WT_W - WT_M, by0 = blockIdx.y * WT_H - WT_M;  // box origin (x a multiple of 4: TMA rule)
    if (tid == 0) {
        q_count = 0;
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(wt_smem_u32(&bar)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(wt_smem_u32(&bar)),
                     "r"((uint32_t)(WB_W * WB_H * sizeof(float))) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
            ::"r"(wt_smem_u32(win)), "l"(reinterpret_cast<uint64_t>(&mapI1)), "r"(bx0), "r"(by0), "r"(wt_smem_u32(&bar))
            : "memory");
    }
    // warp w: columns 32 (w & 1) .. +31 of the tile, rows (w >> 1) + 4 k, k = 0..7 -- a warp's lanes are 32 consecutive
    // pixels of one row, so its taps are (for a smooth flow) consecutive shared-memory words
    const int lx = tid & 63, ly0 = tid >> 6;
    const int x = blockIdx.x * WT_W + lx;
    const int yb = blockIdx.y * WT_H + ly0;
    const bool xin = x < cols;
    float nu1 = 0.f, nu2 = 0.f, nI0 = 0.f;
    if (xin && yb < rows) {
        nu1 = __ldg(&u1p.at(yb, x));
        nu2 = __ldg(&u2p.at(yb, x));
        nI0 = __ldg(&I0.at(yb, x));
    }
    __syncthreads();  // the barrier is initialised before anybody polls it
    wt_mbar_wait(&bar, 0);
#pragma unroll 1
    for (int k = 0; k < WT_H / 4; ++k) {
        const int y = yb + 4 * k;
        const float u1 = nu1, u2 = nu2, I0v = nI0;
        if (k + 1 < WT_H / 4 && xin && y + 4 < rows) {  // next pixel's streaming operands travel under this one's taps
            nu1 = __ldg(&u1p.at(y + 4, x));
            nu2 = __ldg(&u2p.at(y + 4, x));
            nI0 = __ldg(&I0.at(y + 4, x));
        }
        if (!xin || y >= rows) continue;
        int ix, iy;
        float kx[4], ky[4], wsum;
        warp_px_setup(x, y, u1, u2, rows, cols, ix, iy, kx, ky, wsum);
        const int sx = ix - 1 - bx0, sy = iy - 1 - by0;  // the window's top-left tap in box coordinates
        const bool inside = ix >= 1 && iy >= 1 && ix + 4 <= cols - 1 && iy + 4 <= rows - 1;
        if (inside && sx >= 0 && sy >= 0 && sx + 5 < WB_W && sy + 5 < WB_H) {
            float sum, sumx, sumy;
            warp_sep_window<WB_W>(win + sy * WB_W + sx, 0, kx, ky, sum, sumx, sumy);
            warp_px_finish(x, y, u1, u2, I0v, sum, sumx, sumy, wsum, I1wx, I1wy, grad, rho);
        } else {
            q_px[atomicAdd(&q_count, 1)] = (unsigned short)((ly0 + 4 * k) * WT_W + lx);
        }
    }
    __syncthreads();
    const int nq = q_count;
    for (int q = tid; q < nq; q += WT_THREADS) {
        const int e = q_px[q];
        const int qx = blockIdx.x * WT_W + (e & (WT_W - 1)), qy = blockIdx.y * WT_H + (e >> 6);
        const float u1 = __ldg(&u1p.at(qy, qx)), u2 = __ldg(&u2p.at(qy, qx)), I0v = __ldg(&I0.at(qy, qx));
        int ix, iy;
        float kx[4], ky[4], wsum;
        warp_px_setup(qx, qy, u1, u2, rows, cols, ix, iy, kx, ky, wsum);
        const float3 t = warp_slow_taps(I1, rows, cols, ix, iy, kx[0], kx[1], kx[2], kx[3], ky[0], ky[1], ky[2], ky[3]);
        warp_px_finish(qx, qy, u1, u2, I0v, t.x, t.y, t.z, wsum, I1wx, I1wy, grad, rho);
    }
}

// ---------------------------------------------------------------------------------------------
// Unfused, reference-shaped inner iteration (any gamma, optional error image reduction).
// Used for gamma != 0, for the epsilon > 0 cadence and as the cross-check for the blocked kernel.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_tvl1_estimate_u(Tvl1Planes P, int rows, int cols, Tvl1Scalars k,
                                                         int calc_error, double *__restrict__ partials,
                                                         const int *__restrict__ enable) {
    if (enable && __ldg(enable) == 0) return;  // device-side convergence loop: this body does not end with a sample
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    float err = 0.f;
    if (x < cols && y < rows) {
        const float Ix = P.I1wx.at(y, x), Iy = P.I1wy.at(y, x);
        const float g = P.grad.at(y, x), rc = P.rho_c.at(y, x);
        const float u1 = P.u1.at(y, x), u2 = P.u2.at(y, x);
        const float p11 = P.p11.at(y, x), p12 = P.p12.at(y, x);
        const float p21 = P.p21.at(y, x), p22 = P.p22.at(y, x);
        const float p11l = x > 0 ? P.p11.at(y, x - 1) : 0.f;
        const float p21l = x > 0 ? P.p21.at(y, x - 1) : 0.f;
        const float p12u = y > 0 ? P.p12.at(y - 1, x) : 0.f;
        const float p22u = y > 0 ? P.p22.at(y - 1, x) : 0.f;
        float u1n, u2n;
        if (k.gamma == 0.f) {
            tvl1_update_u(k, Ix, Iy, g, rc, u1, u2, p11, p11l, p12, p12u, p21, p21l, p22, p22u, u1n, u2n);
        } else {
            const float u3 = P.u3.at(y, x);
            const float rho = __fadd_rn(rc, __fmaf_rn(k.gamma, u3, __fmaf_rn(Iy, u2, __fmul_rn(Ix, u1))));
            const float fi = tvl1_threshold(rho, g, k.l_t);
            const float v1 = __fmaf_rn(fi, Ix, u1);
            const float v2 = __fmaf_rn(fi, Iy, u2);
            const float v3 = __fmaf_rn(fi, k.gamma, u3);
            const float p31 = P.p31.at(y, x), p32 = P.p32.at(y, x);
            const float p31l = x > 0 ? P.p31.at(y, x - 1) : 0.f;
            const float p32u = y > 0 ? P.p32.at(y - 1, x) : 0.f;
            const float div1 = __fadd_rn(__fsub_rn(p11, p11l), __fsub_rn(p12, p12u));
            const float div2 = __fadd_rn(__fsub_rn(p21, p21l), __fsub_rn(p22, p22u));
            const float div3 = __fadd_rn(__fsub_rn(p31, p31l), __fsub_rn(p32, p32u));
            u1n = __fmaf_rn(k.theta, div1, v1);
            u2n = __fmaf_rn(k.theta, div2, v2);
            P.u3.at(y, x) = __fmaf_rn(k.theta, div3, v3);
        }
        P.u1.at(y, x) = u1n;
        P.u2.at(y, x) = u2n;
        if (calc_error) {
            const float d1 = u1 - u1n, d2 = u2 - u2n;  // u3 is not part of the GPU error (:284-286)
            err = __fmaf_rn(d2, d2, __fmul_rn(d1, d1));
        }
    }
    if (calc_error) {
        // deterministic block reduction in double (the reference uses double atomics, sum.cu:107-133)
        double v = static_cast<double>(err);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        __shared__ double wsum[8];
        const int tid = threadIdx.y * blockDim.x + threadIdx.x;
        if ((tid & 31) == 0) wsum[tid >> 5] = v;
        __syncthreads();
        if (tid == 0) {
            double s = 0.0;
            for (int i = 0; i < 8; ++i) s += wsum[i];
            partials[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
        }
    }
}

__global__ void __launch_bounds__(256) k_tvl1_estimate_dual(Tvl1Planes P, int rows, int cols, Tvl1Scalars k,
                                                            const int *__restrict__ enable) {
    if (enable && __ldg(enable) == 0) return;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const int xr = min(x + 1, cols - 1), yd = min(y + 1, rows - 1);
    {
        const float c1 = P.u1.at(y, x), c2 = P.u2.at(y, x);
        const float ux1 = __fsub_rn(P.u1.at(y, xr), c1), uy1 = __fsub_rn(P.u1.at(yd, x), c1);
        const float ux2 = __fsub_rn(P.u2.at(y, xr), c2), uy2 = __fsub_rn(P.u2.at(yd, x), c2);
        float p11 = P.p11.at(y, x), p12 = P.p12.at(y, x), p21 = P.p21.at(y, x), p22 = P.p22.at(y, x);
        tvl1_update_p2(k.taut, ux1, uy1, ux2, uy2, p11, p12, p21, p22);
        P.p11.at(y, x) = p11;
        P.p12.at(y, x) = p12;
        P.p21.at(y, x) = p21;
        P.p22.at(y, x) = p22;
    }
    if (k.gamma != 0.f) {
        const float c = P.u3.at(y, x);
        const float ux = __fsub_rn(P.u3.at(y, xr), c), uy = __fsub_rn(P.u3.at(yd, x), c);
        float pa = P.p31.at(y, x), pb = P.p32.at(y, x);
        tvl1_update_p(k.taut, ux, uy, pa, pb);
        P.p31.at(y, x) = pa;
        P.p32.at(y, x) = pb;
    }
}

// ---------------------------------------------------------------------------------------------
// cv::medianBlur on the flow planes (float, 3x3 / 5x5, replicated border): the knob of the reference's CPU / OpenCL
// Dual TV-L1 (modules/optflow/src/tvl1flow.cpp:1379-1383, :1266-1269), absent from its CUDA class.  Exact median
// (the reference's float path is a sorting network): partial selection sort of the window up to the middle element.
// Two planes per launch (z = 0: u1, z = 1: u2).
// ---------------------------------------------------------------------------------------------
template <int KS>
__global__ void __launch_bounds__(256) k_tvl1_median(Plane a_in, Plane b_in, Plane a_out, Plane b_out, int rows, int cols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const Plane src = blockIdx.z ? b_in : a_in;
    const Plane dst = blockIdx.z ? b_out : a_out;
    constexpr int R = KS / 2, N = KS * KS;
    float w[N];
#pragma unroll
    for (int j = 0; j < KS; ++j) {
        const int yy = clampi(y + j - R, 0, rows - 1);
#pragma unroll
        for (int i = 0; i < KS; ++i) w[j * KS + i] = __ldg(&src.at(yy, clampi(x + i - R, 0, cols - 1)));
    }
    // the (N/2)-th smallest: after pass k the k smallest sit in w[0..k]
#pragma unroll
    for (int k = 0; k <= N / 2; ++k) {
#pragma unroll
        for (int q = k + 1; q < N; ++q) {
            const float lo = fminf(w[k], w[q]), hi = fmaxf(w[k], w[q]);
            w[k] = lo;
            w[q] = hi;
        }
    }
    dst.at(y, x) = w[N / 2];
}

// Fixed-order final reduction of the per-block partial sums (single block).
__global__ void __launch_bounds__(256) k_reduce_partials(const double *__restrict__ partials, int n,
                                                         double *__restrict__ out, const int *__restrict__ enable) {
    if (enable && __ldg(enable) == 0) return;
    __shared__ double sm[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s += partials[i];
    sm[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sm[0];
}

// ---------------------------------------------------------------------------------------------
// Device-side convergence loop (epsilon > 0).  The reference decides on the HOST, after a blocking copy of the
// error sum, whether to go on (tvl1flow.cpp:357-380); here the same cadence runs on the GPU: the loop is a WHILE
// conditional node of the CUDA graph, its body is
//     [blocked pass A: ia iterations, state set 0 -> 1] [blocked pass B: ib iterations, 1 -> 0]      (unsampled stretch)
//     [estimate_u with error image] [fixed-order reduction] [estimate_dual]                          (sampled iteration)
//     [k_eps_step: book-keeping of the reference's (n, error, prevError), plan of the next body, loop condition]
// with every count read from EpsState at run time (two passes keep the current state set fixed, so every pointer
// in the graph is static; a stretch of m <= 16 unsampled iterations is split ceil(m/2) + floor(m/2), a zero-iteration
// pass B is a plain copy back).  No host synchronisation, no host decision.
// ---------------------------------------------------------------------------------------------
struct EpsState {
    double error, prevError, scaledEps, pe_after;
    int n, iterations;
    int ia, ib;       // iterations of pass A / B of the next body (-1: the body has no unsampled stretch)
    int m;            // ia + ib
    int sample;       // the next body ends with a sampled iteration
    unsigned long long iters_total;  // statistics: iterations run since k_eps_reset
};
enum { EPS_STRETCH_MAX = 16 };

__device__ __forceinline__ void eps_plan(EpsState &s) {
    int m = 0;
    double pe = s.prevError;
    // unsampled iterations ahead: calcError = (n & 1) && prevError < scaledEps; each unsampled one lowers prevError
    while (s.n + m < s.iterations && m < EPS_STRETCH_MAX && !(((s.n + m) & 1) && pe < s.scaledEps)) {
        pe -= s.scaledEps;
        ++m;
    }
    s.m = m;
    s.pe_after = pe;
    s.sample = (s.n + m < s.iterations && ((s.n + m) & 1) && pe < s.scaledEps) ? 1 : 0;
    s.ia = m ? (m + 1) / 2 : -1;
    s.ib = m ? m - (m + 1) / 2 : -1;
}

__global__ void k_eps_reset(EpsState *s) { s->iters_total = 0ull; }

__global__ void k_eps_begin(EpsState *s, double scaledEps, int iterations, cudaGraphConditionalHandle h) {
    s->n = 0;
    s->iterations = iterations;
    s->scaledEps = scaledEps;
    s->prevError = 0.0;                 // tvl1flow.cpp:358
    s->error = 1.7976931348623157e308;  // DBL_MAX
    const bool go = s->error > s->scaledEps && s->n < s->iterations;
    if (go) eps_plan(*s);
    cudaGraphSetConditional(h, go ? 1u : 0u);
}

__global__ void k_eps_step(EpsState *s, const double *__restrict__ err_dev, cudaGraphConditionalHandle h) {
    // account for the body that has just run
    if (s->m) {
        s->n += s->m;
        s->prevError = s->pe_after;
        s->error = 1.7976931348623157e308;
    }
    if (s->sample) {
        s->error = *err_dev;
        s->prevError = s->error;
        s->n += 1;
    }
    s->iters_total += (unsigned long long)(s->m + s->sample);
    const bool go = s->error > s->scaledEps && s->n < s->iterations;
    if (go) eps_plan(*s);
    cudaGraphSetConditional(h, go ? 1u : 0u);
}

// ---------------------------------------------------------------------------------------------
// Host engine
// ---------------------------------------------------------------------------------------------
struct Level {
    int rows = 0, cols = 0;
    Plane I0, I1, u1, u2;
};

class Tvl1Engine : public b2f_handle {
public:
    explicit Tvl1Engine(const b2f_tvl1_params &p) : P(p) { algo = ALGO_TVL1; }
    ~Tvl1Engine() override {
        if (err_host) cudaFreeHost(err_host);
        if (iters_host_) cudaFreeHost(iters_host_);
        free(tma_maps_);
        free(warp_maps_);
    }

    b2f_tvl1_params P;
    // knobs without a counterpart in cv::cuda::OpticalFlowDual_TVL1::create (b2f_set_param only):
    int median_filtering = 1;     // cv::optflow::DualTVL1OpticalFlow::medianFiltering: 1 = off, 3 or 5 = kernel size
    int median_period = 0;        // iterations between two median passes (= the CPU path's innerIterations); 0 = once per warp
    int initial_flow_source = 0;  // useInitialFlow reads: 0 the caller's flow, 1 this handle's previous result (see set_param)

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    const char *default_name() const override { return "DenseOpticalFlow.OpticalFlowDual_TVL1"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"tvl1_iter", "tvl1_warp", "pyramid", "prolong_merge", "reduce"};
        return (cls >= 0 && cls < 5) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        Layout L;
        return layout(rows, cols, true, L);
    }
    bool reads_flow() const override { return P.use_initial_flow != 0 && initial_flow_source == 0; }

private:
    struct Layout {
        std::vector<Level> levels;  // all built levels (the last may be unused, <16 px rule)
        int nscales = 0;            // levels actually solved
        Plane u3[2];                // ping-pong full-res (gamma only)
        float *shared[16] = {};     // level-shared planes, viewed with per-level pitch
        double *partials = nullptr;
        double *err_dev = nullptr;
        EpsState *eps = nullptr;   // device-side convergence loop
        int rows = 0, cols = 0;
        bool gamma = false;
        int nscales_param = 0;
        double scale_step = 0;
    };
    Layout L_;
    double *err_host = nullptr;
    // TMA descriptor blocks, [level][direction], built once per workspace (host memory, 64 B aligned)
    void *tma_maps_ = nullptr;
    bool tma_ok_ = false;
    CUtensorMap *warp_maps_ = nullptr;  // one I1 descriptor per level for the tiled warp kernel; null = not available
    const void *tma_maps(int level, int cur) const {
        return static_cast<const char *>(tma_maps_) + (size_t)(level * 2 + cur) * tvl1_tma_maps_bytes();
    }
    void blocked_planes(int s, Tvl1BlockedPlanes &B) const;

    // graph cache (fixed schedule, or epsilon > 0 on the device loop)
    struct GraphKey {
        int rows, cols;
        b2f_tvl1_params P;
        EngineKnobs knobs;
        int median_filtering, median_period;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && same_knobs(knobs, o.knobs) &&
                   median_filtering == o.median_filtering && median_period == o.median_period && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;

    size_t layout(int rows, int cols, bool counting, Layout &L);
    cudaError_t ensure_workspace(int rows, int cols);
    Plane shared_plane(int idx, int cols) const { return Plane{L_.shared[idx], plane_pitch(cols)}; }
    void solve(Ctx &c, bool allow_sync);
    void proc_one_scale(Ctx &c, int s, Plane &u3cur, bool allow_sync);
    // epsilon > 0 inside a CUDA graph: the reference's adaptive loop as a WHILE conditional node (see EpsState)
    bool device_loop_ok() const {
        return P.epsilon > 0.0 && !L_.gamma && tma_ok_ && knobs.kernel_path == 0 &&
               median_filtering == 1 && !getenv("B2F_TVL1_HOST_LOOP");
    }
    void device_eps_loop(Ctx &c, int s, const Tvl1Planes &T, const Tvl1BlockedPlanes &B, const Tvl1Scalars &k,
                         double scaledEps, dim3 grid, dim3 block, int nblocks, int rows, int cols);
    unsigned long long *iters_host_ = nullptr;  // pinned: EpsState::iters_total of the last device-loop solve
    bool device_loop_used_ = false;
    // active paths: an OR of b2f_tvl1_path flags per solved level
    void mark_path(int s, int flag) { active_paths[s] = static_cast<int>(active_paths[s]) | flag; }
public:
    void refresh_stats() override {
        if (device_loop_used_ && iters_host_) stats.iterations_run = static_cast<int>(*iters_host_);
    }
private:
};

enum { SH_I1WX = 0, SH_I1WY, SH_GRAD, SH_RHO, SH_P11, SH_P12, SH_P21, SH_P22, SH_P31, SH_P32,
       SH_U1B, SH_U2B, SH_P11B, SH_P12B, SH_P21B, SH_P22B, SH_COUNT };

size_t Tvl1Engine::layout(int rows, int cols, bool counting, Layout &L) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.levels.clear();
    L.rows = rows;
    L.cols = cols;
    L.gamma = P.gamma != 0.0;
    L.nscales_param = P.nscales;
    L.scale_step = P.scale_step;
    int r = rows, cc = cols;
    int nscales = P.nscales;
    for (int s = 0; s < P.nscales; ++s) {
        if (s > 0) {
            // cuda::resize dsize rule, resize.cpp:76-79
            r = cv_round(r * P.scale_step);
            cc = cv_round(cc * P.scale_step);
            if (r < 1) r = 1;
            if (cc < 1) cc = 1;
        }
        Level lv;
        lv.rows = r;
        lv.cols = cc;
        lv.I0 = A.plane(r, cc);
        lv.I1 = A.plane(r, cc);
        lv.u1 = A.plane(r, cc);
        lv.u2 = A.plane(r, cc);
        L.levels.push_back(lv);
        if (s > 0 && (cc < 16 || r < 16)) {  // tvl1flow.cpp:243-247
            nscales = s;
            break;
        }
    }
    L.nscales = nscales;
    for (int i = 0; i < SH_COUNT; ++i) {
        if ((i == SH_P31 || i == SH_P32) && !L.gamma) {
            L.shared[i] = nullptr;
            continue;
        }
        L.shared[i] = A.plane(rows, cols).p;
    }
    if (L.gamma) {
        L.u3[0] = A.plane(rows, cols);
        L.u3[1] = A.plane(rows, cols);
    }
    const int nblocks = div_up(cols, 32) * div_up(rows, 8);
    L.partials = static_cast<double *>(A.bytes(sizeof(double) * nblocks));
    L.err_dev = static_cast<double *>(A.bytes(sizeof(double) * 4));
    L.eps = static_cast<EpsState *>(A.bytes(sizeof(EpsState)));
    return A.used();
}

cudaError_t Tvl1Engine::ensure_workspace(int rows, int cols) {
    const bool same = L_.rows == rows && L_.cols == cols && L_.gamma == (P.gamma != 0.0) &&
                      L_.nscales_param == P.nscales && L_.scale_step == P.scale_step && arena.capacity() > 0;
    if (same) return cudaSuccess;
    Layout tmp;
    const size_t need = layout(rows, cols, true, tmp);
    graph_.destroy();
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    layout(rows, cols, false, L_);
    // initial_flow_source 1 starts from a zero field on a fresh workspace
    e = cudaMemset(L_.levels[0].u1.p, 0, sizeof(float) * (size_t)L_.levels[0].u1.pitch * rows);
    if (e == cudaSuccess) e = cudaMemset(L_.levels[0].u2.p, 0, sizeof(float) * (size_t)L_.levels[0].u2.pitch * rows);
    if (e != cudaSuccess) return e;
    if (!err_host) e = cudaMallocHost(&err_host, sizeof(double) * 4);
    if (e != cudaSuccess) return e;
    // TMA descriptors for every solved level and both ping-pong directions
    free(tma_maps_);
    tma_maps_ = nullptr;
    tma_ok_ = false;
    free(warp_maps_);
    warp_maps_ = nullptr;
    if (!getenv("B2F_DISABLE_TMA")) {
        warp_maps_ = static_cast<CUtensorMap *>(aligned_alloc(64, sizeof(CUtensorMap) * (size_t)L_.nscales));
        for (int s = 0; warp_maps_ && s < L_.nscales; ++s) {
            const Level &lv = L_.levels[s];
            if (!tma_encode_2d_f32(&warp_maps_[s], lv.I1.p, (uint64_t)lv.cols, (uint64_t)lv.rows,
                                   (uint64_t)lv.I1.pitch * sizeof(float), WB_W, WB_H)) {
                free(warp_maps_);
                warp_maps_ = nullptr;
            }
        }
    }
    if (!L_.gamma && !getenv("B2F_DISABLE_TMA")) {
        const size_t mb = tvl1_tma_maps_bytes();
        const size_t total = (mb * 2 * L_.nscales + 63) & ~size_t(63);
        tma_maps_ = aligned_alloc(64, total);
        tma_ok_ = tma_maps_ != nullptr;
        for (int s = 0; tma_ok_ && s < L_.nscales; ++s) {
            Tvl1BlockedPlanes B;
            blocked_planes(s, B);
            for (int cur = 0; tma_ok_ && cur < 2; ++cur)
                tma_ok_ = tvl1_tma_build_maps(const_cast<void *>(tma_maps(s, cur)), B, cur, L_.levels[s].rows,
                                              L_.levels[s].cols);
        }
    }
    return cudaSuccess;
}

void Tvl1Engine::blocked_planes(int s, Tvl1BlockedPlanes &B) const {
    const Level &lv = L_.levels[s];
    const int cols = lv.cols;
    B.I1wx = shared_plane(SH_I1WX, cols); B.I1wy = shared_plane(SH_I1WY, cols);
    B.grad = shared_plane(SH_GRAD, cols); B.rho_c = shared_plane(SH_RHO, cols);
    B.s[0].u1 = lv.u1; B.s[0].u2 = lv.u2;
    B.s[0].p11 = shared_plane(SH_P11, cols); B.s[0].p12 = shared_plane(SH_P12, cols);
    B.s[0].p21 = shared_plane(SH_P21, cols); B.s[0].p22 = shared_plane(SH_P22, cols);
    B.s[1].u1 = shared_plane(SH_U1B, cols); B.s[1].u2 = shared_plane(SH_U2B, cols);
    B.s[1].p11 = shared_plane(SH_P11B, cols); B.s[1].p12 = shared_plane(SH_P12B, cols);
    B.s[1].p21 = shared_plane(SH_P21B, cols); B.s[1].p22 = shared_plane(SH_P22B, cols);
}

void Tvl1Engine::device_eps_loop(Ctx &c, int s, const Tvl1Planes &T, const Tvl1BlockedPlanes &B, const Tvl1Scalars &k,
                                 double scaledEps, dim3 grid, dim3 block, int nblocks, int rows, int cols) {
    if (!c.ok()) return;
    cudaStream_t cs = c.stream;  // the capturing stream
    cudaStreamCaptureStatus st;
    cudaGraph_t g = nullptr;
    const cudaGraphNode_t *deps = nullptr;
    size_t nd = 0;
    c.check(cudaStreamGetCaptureInfo_v2(cs, &st, nullptr, &g, &deps, &nd));
    cudaGraphConditionalHandle h;
    if (c.ok()) c.check(cudaGraphConditionalHandleCreate(&h, g, 0, 0));
    if (!c.ok()) return;
    B2F_LAUNCH(c, CLS_REDUCE, 0.0, k_eps_begin, dim3(1), dim3(1), 0, L_.eps, scaledEps, P.iterations, h);
    c.check(cudaStreamGetCaptureInfo_v2(cs, &st, nullptr, &g, &deps, &nd));
    cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
    np.conditional.handle = h;
    np.conditional.type = cudaGraphCondTypeWhile;
    np.conditional.size = 1;
    cudaGraphNode_t node = nullptr;
    if (c.ok()) c.check(cudaGraphAddNode(&node, g, deps, nd, &np));
    if (c.ok()) c.check(cudaStreamUpdateCaptureDependencies(cs, &node, 1, cudaStreamSetCaptureDependencies));
    if (!c.ok()) return;
    cudaGraph_t body = np.conditional.phGraph_out[0];
    cudaStream_t bs = nullptr;
    c.check(cudaStreamCreateWithFlags(&bs, cudaStreamNonBlocking));
    if (!c.ok()) return;
    c.check(cudaStreamBeginCaptureToGraph(bs, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    if (c.ok()) {
        Ctx b = c;
        b.stream = bs;
        const double npx = (double)rows * cols;
        mark_path(s, B2F_TVL1_PATH_ITER_TMA | B2F_TVL1_PATH_ITER_UNFUSED);
        tvl1_tma_launch_dev(b, CLS_ITER, tma_maps(s, 0), B, 0, rows, cols, k, &L_.eps->ia, sm_count());
        tvl1_tma_launch_dev(b, CLS_ITER, tma_maps(s, 1), B, 1, rows, cols, k, &L_.eps->ib, sm_count());
        B2F_LAUNCH(b, CLS_ITER, 48.0 * npx, k_tvl1_estimate_u, grid, block, 0, T, rows, cols, k, 1, L_.partials,
                   &L_.eps->sample);
        B2F_LAUNCH(b, CLS_REDUCE, 8.0 * nblocks, k_reduce_partials, dim3(1), dim3(256), 0, L_.partials, nblocks,
                   L_.err_dev, &L_.eps->sample);
        B2F_LAUNCH(b, CLS_ITER, 40.0 * npx, k_tvl1_estimate_dual, grid, block, 0, T, rows, cols, k, &L_.eps->sample);
        B2F_LAUNCH(b, CLS_REDUCE, 0.0, k_eps_step, dim3(1), dim3(1), 0, L_.eps, L_.err_dev, h);
        c.check(b.err);
        c.check(cudaStreamEndCapture(bs, nullptr));
    }
    cudaStreamDestroy(bs);
}

void Tvl1Engine::proc_one_scale(Ctx &c, int s, Plane &u3cur, bool allow_sync) {
    const Level &lv = L_.levels[s];
    const int rows = lv.rows, cols = lv.cols;
    const double npx = (double)rows * cols;
    const double scaledEpsilon = P.epsilon * P.epsilon * npx;  // tvl1flow.cpp:310
    const bool use_gamma = L_.gamma;

    Tvl1Planes T;
    T.I1wx = shared_plane(SH_I1WX, cols);
    T.I1wy = shared_plane(SH_I1WY, cols);
    T.grad = shared_plane(SH_GRAD, cols);
    T.rho_c = shared_plane(SH_RHO, cols);
    T.p11 = shared_plane(SH_P11, cols);
    T.p12 = shared_plane(SH_P12, cols);
    T.p21 = shared_plane(SH_P21, cols);
    T.p22 = shared_plane(SH_P22, cols);
    T.p31 = use_gamma ? shared_plane(SH_P31, cols) : Plane{nullptr, 0};
    T.p32 = use_gamma ? shared_plane(SH_P32, cols) : Plane{nullptr, 0};
    T.u1 = lv.u1;
    T.u2 = lv.u2;
    T.u3 = use_gamma ? Plane{u3cur.p, plane_pitch(cols)} : Plane{nullptr, 0};

    // p = 0 (tvl1flow.cpp:338-346)
    fill_plane(c, T.p11, rows, cols, 0.f);
    fill_plane(c, T.p12, rows, cols, 0.f);
    fill_plane(c, T.p21, rows, cols, 0.f);
    fill_plane(c, T.p22, rows, cols, 0.f);
    if (use_gamma) {
        fill_plane(c, T.p31, rows, cols, 0.f);
        fill_plane(c, T.p32, rows, cols, 0.f);
    }

    Tvl1Scalars k;
    k.l_t = static_cast<float>(P.lambda * P.theta);  // tvl1flow.cpp:350-351
    k.taut = static_cast<float>(P.tau / P.theta);
    k.theta = static_cast<float>(P.theta);
    k.gamma = static_cast<float>(P.gamma);

    const dim3 block(32, 8);
    const dim3 grid(div_up(cols, 32), div_up(rows, 8));
    const int nblocks = grid.x * grid.y;

    // The temporally blocked kernel needs gamma == 0; with epsilon > 0 it runs the stretches of iterations the
    // reference's cadence does NOT sample (they can never end the loop), the sampled ones go through the
    // unfused kernels with the deterministic error reduction.
    const bool blocked_ok = !use_gamma && knobs.kernel_path != 1;
    Tvl1BlockedPlanes B;
    if (blocked_ok) blocked_planes(s, B);
    const bool use_tma = blocked_ok && tma_ok_ && knobs.kernel_path != 2;
    int cur = 0;  // which state set holds the current (u, p) in the blocked path

    auto point_T_at = [&](int set) {  // unfused kernels work in place on the current state set
        if (!blocked_ok) return;
        T.u1 = B.s[set].u1; T.u2 = B.s[set].u2;
        T.p11 = B.s[set].p11; T.p12 = B.s[set].p12; T.p21 = B.s[set].p21; T.p22 = B.s[set].p22;
    };
    auto run_blocked = [&](int count) {
        int done = 0;
        if (count > 0) mark_path(s, use_tma ? B2F_TVL1_PATH_ITER_TMA : B2F_TVL1_PATH_ITER_BLOCKED);
        while (done < count) {
            const int kk = tvl1_blocked_pick_k(knobs.fused_iters, count - done, rows, cols);
            if (use_tma)  // the persistent TMA kernel
                tvl1_tma_launch(c, CLS_ITER, tma_maps(s, cur), B, cur, rows, cols, k, kk, sm_count());
            else
                tvl1_blocked_launch(c, CLS_ITER, B, cur, rows, cols, k, kk);
            cur ^= 1;
            done += kk;
        }
        c.stats->iterations_run += count;
    };

    // median pass on the current (u1, u2): into the spare state set's planes, then back (the p planes stay put)
    const int med_k = (median_filtering == 3 || median_filtering == 5) ? median_filtering : 1;
    const int med_period = median_period > 0 ? median_period : (P.iterations > 0 ? P.iterations : 1);
    auto median_pass = [&]() {
        point_T_at(cur);
        Plane s1 = blocked_ok ? B.s[cur ^ 1].u1 : shared_plane(SH_U1B, cols);
        Plane s2 = blocked_ok ? B.s[cur ^ 1].u2 : shared_plane(SH_U2B, cols);
        const dim3 gm(grid.x, grid.y, 2);
        if (med_k == 3)
            B2F_LAUNCH(c, CLS_PROLONG, 16.0 * npx, k_tvl1_median<3>, gm, block, 0, T.u1, T.u2, s1, s2, rows, cols);
        else
            B2F_LAUNCH(c, CLS_PROLONG, 16.0 * npx, k_tvl1_median<5>, gm, block, 0, T.u1, T.u2, s1, s2, rows, cols);
        resize_linear_pair(c, CLS_PROLONG, s1, s2, rows, cols, T.u1, T.u2, rows, cols, 1.f, 1.f, 1.f);
    };

    for (int w = 0; w < P.warps; ++w) {
        point_T_at(cur);
        // aux_path 3: the separable kernel on every level (40 registers, 6 blocks / SM; the default before the tiled
        // kernel); any other value: the tiled kernel, levels smaller than one staged box the separable one
        const bool tiled = knobs.aux_path != 3 && warp_maps_ && cols >= WB_W && rows >= WB_H;
        mark_path(s, tiled ? B2F_TVL1_PATH_WARP_TILED : B2F_TVL1_PATH_WARP_UNTILED);
        if (tiled)  // I1 window staged by the copy engine
            B2F_LAUNCH(c, CLS_WARP, 32.0 * npx, k_tvl1_warp_tile<4>, dim3(div_up(cols, WT_W), div_up(rows, WT_H)),
                       dim3(WT_THREADS), 0, warp_maps_[s], lv.I0, lv.I1, T.u1, T.u2, T.I1wx, T.I1wy, T.grad, T.rho_c, rows,
                       cols);
        else
            B2F_LAUNCH(c, CLS_WARP, 32.0 * npx, k_tvl1_warp_sep<6>, grid, block, 0, lv.I0, lv.I1, T.u1, T.u2, T.I1wx,
                       T.I1wy, T.grad, T.rho_c, rows, cols);

        if (blocked_ok && !(P.epsilon > 0.0)) {  // fixed schedule
            if (med_k == 1) {
                run_blocked(P.iterations);
            } else {  // the CPU path's outer loop: median, then `period` inner iterations (tvl1flow.cpp:1377-1404)
                for (int done = 0; done < P.iterations; done += med_period) {
                    median_pass();
                    run_blocked(std::min(med_period, P.iterations - done));
                }
            }
            continue;
        }

        if (c.capturing && device_loop_ok() && blocked_ok && use_tma && cur == 0) {  // same cadence, decided on the GPU
            device_eps_loop(c, s, T, B, k, scaledEpsilon, grid, block, nblocks, rows, cols);
            continue;
        }

        // reference cadence (tvl1flow.cpp:357-380)
        double error = std::numeric_limits<double>::max();
        double prevError = 0.0;
        int n = 0;
        while (error > scaledEpsilon && n < P.iterations) {
            if (med_k > 1 && n % med_period == 0) median_pass();
            const bool calcError = (P.epsilon > 0) && (n & 1) && (prevError < scaledEpsilon);
            if (!calcError && blocked_ok) {
                // count the unsampled iterations ahead (each of them leaves error = DBL_MAX and
                // prevError -= scaledEpsilon) and run them as one blocked stretch
                int m = 0;
                double pe = prevError;
                while (n + m < P.iterations && !((P.epsilon > 0) && ((n + m) & 1) && (pe < scaledEpsilon)) &&
                       !(med_k > 1 && m > 0 && (n + m) % med_period == 0)) {
                    pe -= scaledEpsilon;
                    ++m;
                }
                run_blocked(m);
                prevError = pe;
                error = std::numeric_limits<double>::max();
                n += m;
                continue;
            }
            point_T_at(cur);
            mark_path(s, B2F_TVL1_PATH_ITER_UNFUSED);
            B2F_LAUNCH(c, CLS_ITER, 48.0 * npx, k_tvl1_estimate_u, grid, block, 0, T, rows, cols, k,
                       calcError ? 1 : 0, L_.partials, nullptr);
            if (calcError) {
                B2F_LAUNCH(c, CLS_REDUCE, 8.0 * nblocks, k_reduce_partials, dim3(1), dim3(256), 0, L_.partials,
                           nblocks, L_.err_dev, nullptr);
                if (allow_sync && c.ok()) {
                    c.check(cudaMemcpyAsync(err_host, L_.err_dev, sizeof(double), cudaMemcpyDeviceToHost, c.stream));
                    c.check(cudaStreamSynchronize(c.stream));
                    error = err_host[0];
                    prevError = error;
                }
            } else {
                error = std::numeric_limits<double>::max();
                prevError -= scaledEpsilon;
            }
            B2F_LAUNCH(c, CLS_ITER, 40.0 * npx, k_tvl1_estimate_dual, grid, block, 0, T, rows, cols, k, nullptr);
            c.stats->iterations_run++;
            ++n;
        }
    }

    if (blocked_ok && cur != 0) {
        // the final (u1, u2) live in the B set; the level planes are the A set -> copy back
        resize_linear_pair(c, CLS_PROLONG, B.s[1].u1, B.s[1].u2, rows, cols, lv.u1, lv.u2, rows, cols, 1.f, 1.f, 1.f);
    }
}

void Tvl1Engine::solve(Ctx &c, bool allow_sync) {
    const int ns = L_.nscales;
    if (c.capturing && P.epsilon > 0.0) B2F_LAUNCH(c, CLS_REDUCE, 0.0, k_eps_reset, dim3(1), dim3(1), 0, L_.eps);
    const bool use_gamma = L_.gamma;
    int u3i = 0;
    if (!P.use_initial_flow) {
        fill_plane(c, L_.levels[ns - 1].u1, L_.levels[ns - 1].rows, L_.levels[ns - 1].cols, 0.f);
        fill_plane(c, L_.levels[ns - 1].u2, L_.levels[ns - 1].rows, L_.levels[ns - 1].cols, 0.f);
    }
    if (use_gamma) fill_plane(c, L_.u3[0], L_.rows, L_.cols, 0.f);

    for (int s = ns - 1; s >= 0; --s) {
        proc_one_scale(c, s, L_.u3[u3i], allow_sync);
        if (s == 0) break;
        const Level &lo = L_.levels[s], &hi = L_.levels[s - 1];
        const float inv_fx = inv_scale_from_sizes(lo.cols, hi.cols);
        const float inv_fy = inv_scale_from_sizes(lo.rows, hi.rows);
        const float mul = static_cast<float>(1.0 / P.scale_step);  // tvl1flow.cpp:299-300
        resize_linear_pair(c, CLS_PROLONG, lo.u1, lo.u2, lo.rows, lo.cols, hi.u1, hi.u2, hi.rows, hi.cols, inv_fx,
                           inv_fy, mul);
        if (use_gamma) {  // resized, not rescaled (tvl1flow.cpp:293-296)
            Plane src{L_.u3[u3i].p, plane_pitch(lo.cols)};
            Plane dst{L_.u3[u3i ^ 1].p, plane_pitch(hi.cols)};
            resize_linear_one(c, CLS_PROLONG, src, lo.rows, lo.cols, dst, hi.rows, hi.cols, inv_fx, inv_fy, 1.f);
            u3i ^= 1;
        }
    }
}

int Tvl1Engine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    // preconditions, tvl1flow.cpp:187-191
    if (!(I0->type == B2F_8UC1 || I0->type == B2F_32FC1)) return B2F_UNSUPPORTED_TYPE;
    if (I0->type != I1->type) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    if (P.nscales <= 0) return B2F_BAD_ARG;
    if (P.warps < 0 || P.iterations < 0) return B2F_BAD_ARG;
    if (P.nscales > 1 && !(P.scale_step > 0.0 && P.scale_step < 1.0)) return B2F_BAD_ARG;
    if (!(P.theta > 0.0)) return B2F_BAD_ARG;
    const size_t es = I0->type == B2F_8UC1 ? 1 : 4;
    if (I0->step < I0->cols * es || I1->step < I1->cols * es || !flow_step_ok(flow)) return B2F_BAD_ARG;

    const int rows = I0->rows, cols = I0->cols;
    Ctx c = make_ctx(s);
    tvl1_blocked_init(c);
    c.check(ensure_workspace(rows, cols));
    if (!c.ok()) return finish(c, s);
    stats.levels = L_.nscales;
    stats.iterations_run = 0;
    active_paths.assign(L_.nscales, 0.0);

    const ImageView v0{I0->data, I0->step, rows, cols, I0->type};
    const ImageView v1{I1->data, I1->step, rows, cols, I1->type};
    const ImageView vf = flow_view(flow, rows, cols);

    // convertTo(CV_32F, 8U ? 1 : 255), tvl1flow.cpp:200-201
    convert_pair(c, CLS_PYR, v0, v1, L_.levels[0].I0, L_.levels[0].I1, I0->type == B2F_8UC1 ? 1.0f : 255.0f);
    // initial_flow_source 1: the level-0 planes still hold this handle's previous result (zero after a re-layout)
    if (P.use_initial_flow && initial_flow_source == 0) split_flow(c, CLS_PROLONG, vf, L_.levels[0].u1, L_.levels[0].u2);

    // image (and initial-flow) pyramid, tvl1flow.cpp:238-266
    const int built = static_cast<int>(L_.levels.size());
    for (int l = 1; l < built; ++l) {
        const Level &a = L_.levels[l - 1], &b = L_.levels[l];
        const float inv_f = static_cast<float>(1.0 / P.scale_step);  // fx given -> scale = float(1/fx)
        resize_linear_pair(c, CLS_PYR, a.I0, a.I1, a.rows, a.cols, b.I0, b.I1, b.rows, b.cols, inv_f, inv_f, 1.f);
        if (P.use_initial_flow && l < L_.nscales)
            resize_linear_pair(c, CLS_PROLONG, a.u1, a.u2, a.rows, a.cols, b.u1, b.u2, b.rows, b.cols, inv_f, inv_f,
                               static_cast<float>(P.scale_step));
    }

    const bool fixed_schedule = !(P.epsilon > 0.0);
    const bool dev_loop = !fixed_schedule && device_loop_ok();  // WHILE conditional nodes instead of host decisions
    const bool want_graph = knobs.use_graph && (fixed_schedule || dev_loop) && !profiling && s != nullptr;
    device_loop_used_ = false;
    if (want_graph) {
        const GraphKey key{rows, cols, P, knobs, median_filtering, median_period, L_.levels[0].I0.p};
        if (graph_.run(*this, c, s, key, [&](Ctx &g) { solve(g, false); }) && dev_loop) {
            // the true count lives on the device: fetch it behind the solve, read it in refresh_stats()
            if (!iters_host_) c.check(cudaMallocHost(&iters_host_, sizeof(unsigned long long)));
            if (c.ok())
                c.check(cudaMemcpyAsync(iters_host_, &L_.eps->iters_total, sizeof(unsigned long long),
                                        cudaMemcpyDeviceToHost, s));
            device_loop_used_ = c.ok();
        }
    } else {
        solve(c, true);
    }

    // cuda::merge, tvl1flow.cpp:181-182
    merge_flow(c, CLS_PROLONG, L_.levels[0].u1, L_.levels[0].u2, vf);
    return finish(c, s);
}

int Tvl1Engine::set_param(int id, double v) {
    switch (id) {
        case B2F_TVL1_TAU: P.tau = v; break;
        case B2F_TVL1_LAMBDA: P.lambda = v; break;
        case B2F_TVL1_THETA: P.theta = v; break;
        case B2F_TVL1_NSCALES: P.nscales = static_cast<int>(v); break;
        case B2F_TVL1_WARPS: P.warps = static_cast<int>(v); break;
        case B2F_TVL1_EPSILON: P.epsilon = v; break;
        case B2F_TVL1_ITERATIONS: P.iterations = static_cast<int>(v); break;
        case B2F_TVL1_SCALE_STEP: P.scale_step = v; break;
        case B2F_TVL1_GAMMA: P.gamma = v; break;
        case B2F_TVL1_USE_INITIAL_FLOW: P.use_initial_flow = v != 0; break;
        case B2F_TVL1_MEDIAN_FILTERING: {
            const int k = static_cast<int>(v);
            if (!(k == 1 || k == 3 || k == 5)) return B2F_BAD_ARG;  // cv::medianBlur on CV_32F takes 3 and 5 only
            median_filtering = k;
            break;
        }
        case B2F_TVL1_MEDIAN_PERIOD:
            if (v < 0) return B2F_BAD_ARG;
            median_period = static_cast<int>(v);
            break;
        case B2F_TVL1_INITIAL_FLOW_SOURCE:
            if (!(v == 0 || v == 1)) return B2F_BAD_ARG;
            initial_flow_source = static_cast<int>(v);
            break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

int Tvl1Engine::get_param(int id, double *v) const {
    switch (id) {
        case B2F_TVL1_TAU: *v = P.tau; break;
        case B2F_TVL1_LAMBDA: *v = P.lambda; break;
        case B2F_TVL1_THETA: *v = P.theta; break;
        case B2F_TVL1_NSCALES: *v = P.nscales; break;
        case B2F_TVL1_WARPS: *v = P.warps; break;
        case B2F_TVL1_EPSILON: *v = P.epsilon; break;
        case B2F_TVL1_ITERATIONS: *v = P.iterations; break;
        case B2F_TVL1_SCALE_STEP: *v = P.scale_step; break;
        case B2F_TVL1_GAMMA: *v = P.gamma; break;
        case B2F_TVL1_USE_INITIAL_FLOW: *v = P.use_initial_flow; break;
        case B2F_TVL1_MEDIAN_FILTERING: *v = median_filtering; break;
        case B2F_TVL1_MEDIAN_PERIOD: *v = median_period; break;
        case B2F_TVL1_INITIAL_FLOW_SOURCE: *v = initial_flow_source; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

}  // namespace

}  // namespace b2f

extern "C" {

void b2f_tvl1_default_params(b2f_tvl1_params *p) {
    if (!p) return;
    p->tau = 0.25;
    p->lambda = 0.15;
    p->theta = 0.3;
    p->nscales = 5;
    p->warps = 5;
    p->epsilon = 0.01;
    p->iterations = 300;
    p->scale_step = 0.8;
    p->gamma = 0.0;
    p->use_initial_flow = 0;
}

int b2f_median_blur_32f(const b2f_image *src, b2f_image *dst, int ksize, void *cuda_stream) {
    using namespace b2f;
    if (!src || !dst || !src->data || !dst->data) return B2F_BAD_ARG;
    if (src->type != B2F_32FC1 || dst->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
    if (src->rows != dst->rows || src->cols != dst->cols) return B2F_SIZE_MISMATCH;
    if (!(ksize == 3 || ksize == 5) || src->rows <= 0 || src->cols <= 0 || (src->step % 4) || (dst->step % 4) ||
        src->step < (size_t)src->cols * 4 || dst->step < (size_t)dst->cols * 4 || src->data == dst->data)
        return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(src->data, s);
    const Plane a{static_cast<float *>(src->data), (int)(src->step / 4)}, b{static_cast<float *>(dst->data), (int)(dst->step / 4)};
    const dim3 block(32, 8), grid(div_up(src->cols, 32), div_up(src->rows, 8), 1);
    if (ksize == 3) k_tvl1_median<3><<<grid, block, 0, s>>>(a, a, b, b, src->rows, src->cols);
    else k_tvl1_median<5><<<grid, block, 0, s>>>(a, a, b, b, src->rows, src->cols);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && s == nullptr) e = cudaDeviceSynchronize();
    return e == cudaSuccess ? B2F_OK : B2F_CUDA_ERROR;
}

int b2f_tvl1_create(const b2f_tvl1_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_tvl1_params d;
    b2f_tvl1_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::Tvl1Engine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
