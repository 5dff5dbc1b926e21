// tvl1_math.cuh -- the per-pixel arithmetic of the Dual TV-L1 inner loop, written once with
// explicit rounding intrinsics so that every kernel variant (unfused, fused, temporally blocked)
// produces bit-identical values for the same inputs regardless of how ptxas would otherwise
// contract mul+add pairs.  Semantics follow the reference kernels:
//   estimateUKernel             modules/cudaoptflow/src/cuda/tvl1flow.cu:209-288
//   estimateDualVariablesKernel modules/cudaoptflow/src/cuda/tvl1flow.cu:313-348
// Deliberate arithmetic choices (documented in DESIGN.md; oracle/tvl1_gpu_model.c built with -DENGINE_ROUNDING restates
// each of them, and the engine equals that model bit for bit in tests/test_tvl1_gpu.py and test_tvl1_fullsize_gpu.py,
// rcp.approx / sqrt.approx emulated from tables of the device's own values):
//   * -rho/grad is -rho * rcp.approx(grad) (MUFU.RCP, <= 2 ulp) instead of an IEEE divide, and the
//     three-way threshold test is written as the equivalent clamp (see tvl1_threshold);
//   * hypotf(a,b) is sqrt.approx(a*a + b*b) and the dual normalisation multiplies by a shared
//     rcp.approx instead of IEEE divides (see tvl1_update_p2);
//   * the divergence at the first row/column uses a zero ghost value, (p - 0) + (q - q_up), where
//     the reference writes p + q - q_up: same value up to one rounding on that column only.
#pragma once
#include "common.cuh"

namespace b2f {

struct Tvl1Scalars {
    float l_t;    // lambda * theta
    float theta;  // theta
    float taut;   // tau / theta
    float gamma;  // illumination weight (0 = off)
};

#ifdef __CUDACC__

// Per-pixel constant of the thresholding step: 1/|grad I|^2, or a huge value where the reference
// treats the gradient as zero (grad <= FLT_EPSILON), so that the clamp below degenerates to the
// reference's sign test there.  Constant over the inner iterations of a warp: the warp kernels
// evaluate it once per pixel and store it in the `grad` plane.
__device__ __forceinline__ float tvl1_inv_grad(float grad) { return grad > FLT_EPSILON ? rcp_approx(grad) : 1e30f; }

// Thresholding step TH (tvl1flow.cu:236-262): the multiplier fi with d = fi * (Ix, Iy, gamma).
// The reference's three-way test  rho < -l_t*g -> l_t ; rho > l_t*g -> -l_t ; else -rho/g  is the
// clamp of -rho/g to [-l_t, l_t] (TH is continuous in rho), evaluated branch-free with two FMNMX.
__device__ __forceinline__ float tvl1_threshold(float rho, float inv_grad, float l_t) {
    return fminf(fmaxf(__fmul_rn(-rho, inv_grad), -l_t), l_t);
}

// One primal update for a single pixel.  pl = p11(x-1) (0 at x==0), pu = p12(y-1) (0 at y==0).
__device__ __forceinline__ void tvl1_update_u(const Tvl1Scalars &k, float Ix, float Iy, float inv_grad, float rho_c,
                                              float u1, float u2, float p11, float p11_l, float p12, float p12_u,
                                              float p21, float p21_l, float p22, float p22_u, float &u1n,
                                              float &u2n) {
    const float rho = __fmaf_rn(Iy, u2, __fmaf_rn(Ix, u1, rho_c));  // two FMAs (the reference's nvcc build contracts too)
    const float fi = tvl1_threshold(rho, inv_grad, k.l_t);
    const float v1 = __fmaf_rn(fi, Ix, u1);
    const float v2 = __fmaf_rn(fi, Iy, u2);
    const float div1 = __fadd_rn(__fsub_rn(p11, p11_l), __fsub_rn(p12, p12_u));
    const float div2 = __fadd_rn(__fsub_rn(p21, p21_l), __fsub_rn(p22, p22_u));
    u1n = __fmaf_rn(k.theta, div1, v1);
    u2n = __fmaf_rn(k.theta, div2, v2);
}

// Dual update of both flow components of one pixel (estimateDualVariablesKernel, tvl1flow.cu:313-348).
// ux*, uy* are the forward differences (0 on the last column / row).  The two normalisations
// 1/(1 + taut*g1), 1/(1 + taut*g2) share ONE reciprocal: r = 1/(a1*a2), inv1 = r*a2, inv2 = r*a1 (a1, a2 >= 1).
// The SFU path (16 lanes/SM, fed through the MIO queue together with LDS / STS / SHFL) is the first thing
// to saturate in the dual half iteration, so three FMULs are preferred over a fourth MUFU per pixel.
__device__ __forceinline__ void tvl1_update_p2(float taut, float ux1, float uy1, float ux2, float uy2, float &p11,
                                               float &p12, float &p21, float &p22) {
    const float g1 = sqrt_approx(__fmaf_rn(ux1, ux1, __fmul_rn(uy1, uy1)));
    const float g2 = sqrt_approx(__fmaf_rn(ux2, ux2, __fmul_rn(uy2, uy2)));
    const float a1 = __fmaf_rn(taut, g1, 1.0f);
    const float a2 = __fmaf_rn(taut, g2, 1.0f);
    const float r = rcp_approx(__fmul_rn(a1, a2));
    const float inv1 = __fmul_rn(r, a2), inv2 = __fmul_rn(r, a1);
    p11 = __fmul_rn(__fmaf_rn(taut, ux1, p11), inv1);
    p12 = __fmul_rn(__fmaf_rn(taut, uy1, p12), inv1);
    p21 = __fmul_rn(__fmaf_rn(taut, ux2, p21), inv2);
    p22 = __fmul_rn(__fmaf_rn(taut, uy2, p22), inv2);
}

// Single-component dual update (third, illumination component when gamma != 0).
__device__ __forceinline__ void tvl1_update_p(float taut, float ux, float uy, float &pa, float &pb) {
    const float g = sqrt_approx(__fmaf_rn(ux, ux, __fmul_rn(uy, uy)));
    const float inv = rcp_approx(__fmaf_rn(taut, g, 1.0f));
    pa = __fmul_rn(__fmaf_rn(taut, ux, pa), inv);
    pb = __fmul_rn(__fmaf_rn(taut, uy, pb), inv);
}

#endif  // __CUDACC__

}  // namespace b2f
