// sparselk.cu -- cv::cuda::SparsePyrLKOpticalFlow (SURVEY.md 8f rank 4): pyramidal Lucas-Kanade for a list of
// points, the sparse sibling of DensePyrLK that videostab uses (modules/videostab/src/optical_flow.cpp:105-111).
//
// Reference: modules/cudaoptflow/src/pyrlk.cpp:153-236 (driver), src/cuda/pyrlk.cu:148-345 (sparseKernel):
//   * pyramid by cuda::pyrDown on the INPUT type (8-bit levels are rounded, pyr_down.cu:172);
//   * nextPts starts at prevPts (or the caller's estimate) / 2^(maxLevel+1)  (pyrlk.cpp:168-170);
//   * per level, one 16x16 block per point: bilinear patch of I and its Scharr derivatives around
//     prevPt / 2^level, the 2x2 covariance by a block reduction, up to `iters` Newton steps on J, then
//     nextPts[i] = nextPt; a point that leaves the image or has a singular matrix returns early WITHOUT
//     updating nextPts, and clears status only on level 0 (pyrlk.cu:162-168,232-238,256-262);
//   * 8-bit images are read through normalised-float textures (values / 255), so the error output is
//     scaled back by 255 (DenormalizationFactor, :139-146).
// Types: every instantiation of the reference's dispatcher table (pyrlk.cpp:195-203): 8U / 16U / 32S / 32F with 1, 3 or
// 4 channels.  The reference runs them through TWO sampling paths, reproduced here as SAMP_TEX / SAMP_SOFT:
//   texture path  (8UC1, 8UC4, 16UC4, 32FC1, 32FC4; sparseKernel :148-345): hardware bilinear with 8-bit weights, clamp
//                 addressing, integer texels read as normalised floats (value / 255, value / 65535);
//   software path (every 3-channel type, 16UC1, 32SC1, 32SC4; sparseKernel_ :343-534, sparse_caller specialisations
//                 :575-700): LinearFilter<BorderReader<BrdConstant>> of opencv core (cuda/filters.hpp, external to
//                 opencv_contrib): exact float weights from floor(x), zero outside the image, raw (unnormalised) values,
//                 and the bilinear result is saturate_cast back to the element type (rounded for integer depths).
// The A / b sums run over ALL channels (accum, :66-81), the error divides by min(cn, 3) (:341,:528).
// CV_8UC1 and CV_32FC1 keep their dedicated single-plane kernel (k_sparse_lk); everything else uses k_sparse_lk_mc.
// Oracle: cv2.calcOpticalFlowPyrLK with the reference's own criterion (test_optflow.cpp:241-264).
#include <cstring>
#include <new>

#include "common.cuh"

struct b2f_sparse {
    b2f_sparselk_params P;
    b2f::Arena arena;
    int rows = 0, cols = 0, levels = 0, planes = 0;  // planes = channels held per image (I / J hold levels * planes)
    std::vector<b2f::Plane> I, J;
    std::vector<int> lrows, lcols;
    int last_cuda_error = 0;
    b2f_stats stats{};
};

namespace b2f {
namespace {

constexpr int SB = 256;  // 16 x 16 threads per point (pyrlk.cpp:116-133 calcPatchSize, compute >= 1.2)
constexpr int RED = 3 * (SB / 32);  // block_sum's staging (`red`): the kernels' only static shared memory
constexpr size_t STATIC_SMEM = RED * sizeof(float);

struct TexView {
    Plane p;
    int rows, cols;
    float inv_norm;  // 1 for float images; 8-bit images are fetched as value / 255
};

__device__ __forceinline__ float sp_texel(const TexView &t, int y, int x) {
    const float v = __ldg(&t.p.at(clampi(y, 0, t.rows - 1), clampi(x, 0, t.cols - 1)));
    return t.inv_norm == 1.f ? v : __fdiv_rn(v, 255.f);
}

// unnormalised coordinates, linear filter with 8-bit weights, clamp addressing (TextureLinear, pyrlk.cu:535-554)
__device__ __forceinline__ float sp_tex(const TexView &t, float y, float x) {
    const float xb = x - 0.5f, yb = y - 0.5f;
    const float fx = floorf(xb), fy = floorf(yb);
    const float ax = floorf((xb - fx) * 256.f + 0.5f) * (1.f / 256.f);
    const float ay = floorf((yb - fy) * 256.f + 0.5f) * (1.f / 256.f);
    const int x0 = (int)fminf(fmaxf(fx, -2.f), (float)t.cols + 1.f), y0 = (int)fminf(fmaxf(fy, -2.f), (float)t.rows + 1.f);
    const float t00 = sp_texel(t, y0, x0), t01 = sp_texel(t, y0, x0 + 1);
    const float t10 = sp_texel(t, y0 + 1, x0), t11 = sp_texel(t, y0 + 1, x0 + 1);
    return (1.f - ax) * (1.f - ay) * t00 + ax * (1.f - ay) * t01 + (1.f - ax) * ay * t10 + ax * ay * t11;
}

// deterministic block sum of up to three values; every thread receives the totals
template <int N>
__device__ __forceinline__ void block_sum(float (&v)[N], float *red /* N * 8 floats */, int tid) {
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
    __syncthreads();  // protects `red` from the previous use
    if ((tid & 31) == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) red[k * 8 + (tid >> 5)] = v[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        float s = red[k * 8];
#pragma unroll
        for (int w = 1; w < SB / 32; ++w) s += red[k * 8 + w];
        v[k] = s;
    }
}

__global__ void __launch_bounds__(SB) k_sparse_lk(TexView I, TexView J, const float2 *__restrict__ prevPts,
                                                   float2 *__restrict__ nextPts, unsigned char *__restrict__ status,
                                                   float *__restrict__ err, int level, int win_x, int win_y, int half_x,
                                                   int half_y, int iters, float err_scale) {
    extern __shared__ float sp_smem[];
    const int n_win = win_x * win_y;
    float *I_patch = sp_smem, *dIdx_patch = sp_smem + n_win, *dIdy_patch = sp_smem + 2 * n_win;
    __shared__ float red[RED];
    const int tid = threadIdx.x;
    const int pt = blockIdx.x;
    const int rows = I.rows, cols = I.cols;

    float2 prevPt = prevPts[pt];
    prevPt.x *= (1.0f / (1 << level));
    prevPt.y *= (1.0f / (1 << level));
    if (prevPt.x < 0 || prevPt.x >= cols || prevPt.y < 0 || prevPt.y >= rows) {
        if (tid == 0 && level == 0) status[pt] = 0;
        return;
    }
    prevPt.x -= half_x;
    prevPt.y -= half_y;

    float a[3] = {0.f, 0.f, 0.f};
    for (int e = tid; e < n_win; e += SB) {
        const int yB = e / win_x, xB = e - yB * win_x;
        const float x = prevPt.x + xB + 0.5f, y = prevPt.y + yB + 0.5f;
        I_patch[e] = sp_tex(I, y, x);
        const float dx = 3.0f * sp_tex(I, y - 1, x + 1) + 10.0f * sp_tex(I, y, x + 1) + 3.0f * sp_tex(I, y + 1, x + 1) -
                         (3.0f * sp_tex(I, y - 1, x - 1) + 10.0f * sp_tex(I, y, x - 1) + 3.0f * sp_tex(I, y + 1, x - 1));
        const float dy = 3.0f * sp_tex(I, y + 1, x - 1) + 10.0f * sp_tex(I, y + 1, x) + 3.0f * sp_tex(I, y + 1, x + 1) -
                         (3.0f * sp_tex(I, y - 1, x - 1) + 10.0f * sp_tex(I, y - 1, x) + 3.0f * sp_tex(I, y - 1, x + 1));
        dIdx_patch[e] = dx;
        dIdy_patch[e] = dy;
        a[0] += dx * dx;
        a[1] += dx * dy;
        a[2] += dy * dy;
    }
    block_sum<3>(a, red, tid);
    float A11 = a[0], A12 = a[1], A22 = a[2];
    float D = A11 * A22 - A12 * A12;
    if (D < FLT_EPSILON) {
        if (tid == 0 && level == 0) status[pt] = 0;
        return;
    }
    D = 1.f / D;
    A11 *= D;
    A12 *= D;
    A22 *= D;

    float2 nextPt = nextPts[pt];
    nextPt.x *= 2.f;
    nextPt.y *= 2.f;
    nextPt.x -= half_x;
    nextPt.y -= half_y;

    for (int k = 0; k < iters; ++k) {
        if (nextPt.x < -half_x || nextPt.x >= cols || nextPt.y < -half_y || nextPt.y >= rows) {
            if (tid == 0 && level == 0) status[pt] = 0;
            return;
        }
        float b[2] = {0.f, 0.f};
        for (int e = tid; e < n_win; e += SB) {
            const int yB = e / win_x, xB = e - yB * win_x;
            const float Jv = sp_tex(J, nextPt.y + yB + 0.5f, nextPt.x + xB + 0.5f);
            const float diff = (Jv - I_patch[e]) * 32.0f;
            b[0] += diff * dIdx_patch[e];
            b[1] += diff * dIdy_patch[e];
        }
        block_sum<2>(b, red, tid);
        const float dx = A12 * b[1] - A22 * b[0];
        const float dy = A12 * b[0] - A11 * b[1];
        nextPt.x += dx;
        nextPt.y += dy;
        if (fabsf(dx) < 0.01f && fabsf(dy) < 0.01f) break;
    }

    float ev[1] = {0.f};
    if (err != nullptr) {
        for (int e = tid; e < n_win; e += SB) {
            const int yB = e / win_x, xB = e - yB * win_x;
            const float Jv = sp_tex(J, nextPt.y + yB + 0.5f, nextPt.x + xB + 0.5f);
            ev[0] += fabsf(Jv - I_patch[e]);
        }
        block_sum<1>(ev, red, tid);
    }
    if (tid == 0) {
        nextPt.x += half_x;
        nextPt.y += half_y;
        nextPts[pt] = nextPt;
        if (err != nullptr) err[pt] = ev[0] / (float)(win_x * win_y) * err_scale;  // cn = 1 (pyrlk.cu:341)
    }
}

// ---------------------------------------------------------------------------------------------
// multi-channel / multi-depth variant
// ---------------------------------------------------------------------------------------------
constexpr int MAXC = 4;
struct TexViewN {
    Plane p[MAXC];
    int rows, cols;
    float norm;     // SAMP_TEX: texels are divided by this (255, 65535 or 1: cudaReadModeNormalizedFloat)
    float lo, hi;   // SAMP_SOFT: saturate_cast range of the element type (lo > hi: float, no rounding)
};
enum { SAMP_TEX = 0, SAMP_SOFT = 1 };

template <int CN, int SAMP>
__device__ __forceinline__ void spn_sample(const TexViewN &t, float y, float x, float (&out)[CN]) {
    if (SAMP == SAMP_TEX) {
        const float xb = x - 0.5f, yb = y - 0.5f;
        const float fx = floorf(xb), fy = floorf(yb);
        const float ax = floorf((xb - fx) * 256.f + 0.5f) * (1.f / 256.f);
        const float ay = floorf((yb - fy) * 256.f + 0.5f) * (1.f / 256.f);
        const int x0 = (int)fminf(fmaxf(fx, -2.f), (float)t.cols + 1.f), y0 = (int)fminf(fmaxf(fy, -2.f), (float)t.rows + 1.f);
        const int xa = clampi(x0, 0, t.cols - 1), xb2 = clampi(x0 + 1, 0, t.cols - 1);
        const int ya = clampi(y0, 0, t.rows - 1), yb2 = clampi(y0 + 1, 0, t.rows - 1);
#pragma unroll
        for (int c = 0; c < CN; ++c) {
            const float t00 = __fdiv_rn(__ldg(&t.p[c].at(ya, xa)), t.norm), t01 = __fdiv_rn(__ldg(&t.p[c].at(ya, xb2)), t.norm);
            const float t10 = __fdiv_rn(__ldg(&t.p[c].at(yb2, xa)), t.norm), t11 = __fdiv_rn(__ldg(&t.p[c].at(yb2, xb2)), t.norm);
            out[c] = (1.f - ax) * (1.f - ay) * t00 + ax * (1.f - ay) * t01 + (1.f - ax) * ay * t10 + ax * ay * t11;
        }
    } else {
        const float fx = floorf(fminf(fmaxf(x, -4.f), (float)t.cols + 4.f)), fy = floorf(fminf(fmaxf(y, -4.f), (float)t.rows + 4.f));
        const int x1 = (int)fx, y1 = (int)fy, x2 = x1 + 1, y2 = y1 + 1;
        const float w11 = ((float)x2 - x) * ((float)y2 - y), w12 = (x - (float)x1) * ((float)y2 - y);
        const float w21 = ((float)x2 - x) * (y - (float)y1), w22 = (x - (float)x1) * (y - (float)y1);
        const bool r1 = y1 >= 0 && y1 < t.rows, r2 = y2 >= 0 && y2 < t.rows;
        const bool c1 = x1 >= 0 && x1 < t.cols, c2 = x2 >= 0 && x2 < t.cols;
#pragma unroll
        for (int c = 0; c < CN; ++c) {
            float o = 0.f;
            o = o + (r1 && c1 ? __ldg(&t.p[c].at(y1, x1)) : 0.f) * w11;
            o = o + (r1 && c2 ? __ldg(&t.p[c].at(y1, x2)) : 0.f) * w12;
            o = o + (r2 && c1 ? __ldg(&t.p[c].at(y2, x1)) : 0.f) * w21;
            o = o + (r2 && c2 ? __ldg(&t.p[c].at(y2, x2)) : 0.f) * w22;
            out[c] = t.lo > t.hi ? o : rintf(fminf(fmaxf(o, t.lo), t.hi));  // saturate_cast<elem_type>
        }
    }
}

template <int CN, int SAMP>
__global__ void __launch_bounds__(SB) k_sparse_lk_mc(TexViewN I, TexViewN J, const float2 *__restrict__ prevPts,
                                                      float2 *__restrict__ nextPts, unsigned char *__restrict__ status,
                                                      float *__restrict__ err, int level, int win_x, int win_y, int half_x,
                                                      int half_y, int iters, float err_scale) {
    extern __shared__ float sp_smem[];
    const int n_win = win_x * win_y;
    float *I_patch = sp_smem, *dIdx_patch = sp_smem + CN * n_win, *dIdy_patch = sp_smem + 2 * CN * n_win;
    __shared__ float red[RED];
    const int tid = threadIdx.x;
    const int pt = blockIdx.x;
    const int rows = I.rows, cols = I.cols;

    float2 prevPt = prevPts[pt];
    prevPt.x *= (1.0f / (1 << level));
    prevPt.y *= (1.0f / (1 << level));
    if (prevPt.x < 0 || prevPt.x >= cols || prevPt.y < 0 || prevPt.y >= rows) {
        if (tid == 0 && level == 0) status[pt] = 0;
        return;
    }
    prevPt.x -= half_x;
    prevPt.y -= half_y;

    float a[3] = {0.f, 0.f, 0.f};
    for (int e = tid; e < n_win; e += SB) {
        const int yB = e / win_x, xB = e - yB * win_x;
        const float x = prevPt.x + xB + 0.5f, y = prevPt.y + yB + 0.5f;
        float v[CN], mm[CN], m0[CN], mp[CN], zm[CN], zp[CN], pm[CN], p0[CN], pp[CN];
        spn_sample<CN, SAMP>(I, y, x, v);
        spn_sample<CN, SAMP>(I, y - 1, x - 1, mm); spn_sample<CN, SAMP>(I, y - 1, x, m0); spn_sample<CN, SAMP>(I, y - 1, x + 1, mp);
        spn_sample<CN, SAMP>(I, y, x - 1, zm); spn_sample<CN, SAMP>(I, y, x + 1, zp);
        spn_sample<CN, SAMP>(I, y + 1, x - 1, pm); spn_sample<CN, SAMP>(I, y + 1, x, p0); spn_sample<CN, SAMP>(I, y + 1, x + 1, pp);
#pragma unroll
        for (int c = 0; c < CN; ++c) {
            const float dx = 3.0f * mp[c] + 10.0f * zp[c] + 3.0f * pp[c] - (3.0f * mm[c] + 10.0f * zm[c] + 3.0f * pm[c]);
            const float dy = 3.0f * pm[c] + 10.0f * p0[c] + 3.0f * pp[c] - (3.0f * mm[c] + 10.0f * m0[c] + 3.0f * mp[c]);
            I_patch[c * n_win + e] = v[c];
            dIdx_patch[c * n_win + e] = dx;
            dIdy_patch[c * n_win + e] = dy;
            a[0] += dx * dx;
            a[1] += dx * dy;
            a[2] += dy * dy;
        }
    }
    block_sum<3>(a, red, tid);
    float A11 = a[0], A12 = a[1], A22 = a[2];
    float D = A11 * A22 - A12 * A12;
    if (D < FLT_EPSILON) {
        if (tid == 0 && level == 0) status[pt] = 0;
        return;
    }
    D = 1.f / D;
    A11 *= D;
    A12 *= D;
    A22 *= D;

    float2 nextPt = nextPts[pt];
    nextPt.x *= 2.f;
    nextPt.y *= 2.f;
    nextPt.x -= half_x;
    nextPt.y -= half_y;

    for (int k = 0; k < iters; ++k) {
        if (nextPt.x < -half_x || nextPt.x >= cols || nextPt.y < -half_y || nextPt.y >= rows) {
            if (tid == 0 && level == 0) status[pt] = 0;
            return;
        }
        float b[2] = {0.f, 0.f};
        for (int e = tid; e < n_win; e += SB) {
            const int yB = e / win_x, xB = e - yB * win_x;
            float Jv[CN];
            spn_sample<CN, SAMP>(J, nextPt.y + yB + 0.5f, nextPt.x + xB + 0.5f, Jv);
#pragma unroll
            for (int c = 0; c < CN; ++c) {
                const float diff = (Jv[c] - I_patch[c * n_win + e]) * 32.0f;
                b[0] += diff * dIdx_patch[c * n_win + e];
                b[1] += diff * dIdy_patch[c * n_win + e];
            }
        }
        block_sum<2>(b, red, tid);
        const float dx = A12 * b[1] - A22 * b[0];
        const float dy = A12 * b[0] - A11 * b[1];
        nextPt.x += dx;
        nextPt.y += dy;
        if (fabsf(dx) < 0.01f && fabsf(dy) < 0.01f) break;
    }

    float ev[1] = {0.f};
    if (err != nullptr) {
        for (int e = tid; e < n_win; e += SB) {
            const int yB = e / win_x, xB = e - yB * win_x;
            float Jv[CN];
            spn_sample<CN, SAMP>(J, nextPt.y + yB + 0.5f, nextPt.x + xB + 0.5f, Jv);
#pragma unroll
            for (int c = 0; c < CN; ++c) ev[0] += fabsf(Jv[c] - I_patch[c * n_win + e]);
        }
        block_sum<1>(ev, red, tid);
    }
    if (tid == 0) {
        nextPt.x += half_x;
        nextPt.y += half_y;
        nextPts[pt] = nextPt;
        if (err != nullptr) err[pt] = ev[0] / (float)((CN < 3 ? CN : 3) * win_x * win_y) * err_scale;  // :341 / :528
    }
}

// interleaved T x CN image (byte pitch) -> CN float planes, both frames per launch (z = frame)
template <typename T>
__global__ void __launch_bounds__(256) k_sparse_deinterleave(const T *__restrict__ a, const T *__restrict__ b, size_t step_a,
                                                             size_t step_b, TexViewN da, TexViewN db, int cn) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= da.cols || y >= da.rows) return;
    const T *src = reinterpret_cast<const T *>(reinterpret_cast<const char *>(blockIdx.z ? b : a) + (size_t)y * (blockIdx.z ? step_b : step_a));
    const TexViewN &d = blockIdx.z ? db : da;
    for (int c = 0; c < cn; ++c) d.p[c].at(y, x) = static_cast<float>(src[(size_t)x * cn + c]);
}

// cv::cuda::pyrDown of one plane with the element type's saturate_cast (round half to even, clamp) applied to the result
__global__ void __launch_bounds__(256) k_sparse_quantize(Plane d, int rows, int cols, float lo, float hi) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    d.at(y, x) = rintf(fminf(fmaxf(d.at(y, x), lo), hi));
}

__global__ void k_sparse_init(const float2 *__restrict__ src, float2 *__restrict__ dst, unsigned char *__restrict__ status,
                              int n, float scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 p = src[i];
    dst[i] = make_float2(p.x * scale, p.y * scale);  // cuda::multiply(pts, 1 / 2^(maxLevel+1)), pyrlk.cpp:168-170
    status[i] = 1;                                    // status.setTo(1), :173-174
}

// cudaDevAttrMaxSharedMemoryPerBlockOptin of the current device, queried once per device; 0 when the query fails
int smem_optin_limit() {
    constexpr int kMaxDevices = 64;
    static std::atomic<int> cache[kMaxDevices] = {};
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    const bool tracked = dev >= 0 && dev < kMaxDevices;
    if (tracked) {
        const int v = cache[dev].load(std::memory_order_relaxed);
        if (v > 0) return v;
    }
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    if (tracked) cache[dev].store(v, std::memory_order_relaxed);
    return v;
}

bool aligned(const void *p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a == 0; }

}  // namespace
}  // namespace b2f

extern "C" {

void b2f_sparselk_default_params(b2f_sparselk_params *p) {
    if (!p) return;
    p->win_width = 21;  // cudaoptflow.hpp:221-225
    p->win_height = 21;
    p->max_level = 3;
    p->iters = 30;
    p->use_initial_flow = 0;
}

int b2f_sparselk_create(const b2f_sparselk_params *p, b2f_sparse **out) {
    if (!out) return B2F_BAD_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return B2F_NO_DEVICE;
    }
    b2f_sparse *h = new (std::nothrow) b2f_sparse;
    if (!h) return B2F_OUT_OF_MEMORY;
    if (p) h->P = *p; else b2f_sparselk_default_params(&h->P);
    *out = h;
    return B2F_OK;
}

void b2f_sparselk_destroy(b2f_sparse *h) { delete h; }

int b2f_sparselk_set_params(b2f_sparse *h, const b2f_sparselk_params *p) {
    if (!h || !p) return B2F_BAD_ARG;
    h->P = *p;
    return B2F_OK;
}
int b2f_sparselk_get_params(const b2f_sparse *h, b2f_sparselk_params *p) {
    if (!h || !p) return B2F_BAD_ARG;
    *p = h->P;
    return B2F_OK;
}

int b2f_sparselk_calc(b2f_sparse *h, const b2f_image *prev_img, const b2f_image *next_img, const float *prev_pts,
                      float *next_pts, unsigned char *status, float *err, int n_points, void *cuda_stream) {
    using namespace b2f;
    if (!h || !prev_img || !next_img || !prev_img->data || !next_img->data) return B2F_BAD_ARG;
    if (n_points < 0) return B2F_BAD_ARG;
    if (n_points == 0) return B2F_OK;  // pyrlk.cpp:221-227: empty input, empty output
    if (!prev_pts || !next_pts || !status) return B2F_BAD_ARG;
    const b2f_sparselk_params &P = h->P;
    const int depth = prev_img->type & 7, cn = (prev_img->type >> 3) + 1;
    if (prev_img->type < 0 || prev_img->type > 31) return B2F_UNSUPPORTED_TYPE;
    if (!(depth == 0 || depth == 2 || depth == 4 || depth == 5) || !(cn == 1 || cn == 3 || cn == 4))
        return B2F_UNSUPPORTED_TYPE;  // funcs[][] table + CV_Assert(channels 1 / 3 / 4), pyrlk.cpp:195-206,228
    if (next_img->type != prev_img->type) return B2F_UNSUPPORTED_TYPE;                                 // pyrlk.cpp:229
    if (prev_img->rows != next_img->rows || prev_img->cols != next_img->cols) return B2F_SIZE_MISMATCH;
    if (P.max_level < 0 || !(P.win_width > 2 && P.win_height > 2) || P.iters < 0) return B2F_BAD_ARG;  // :160-161
    if (P.max_level > 30) return B2F_BAD_ARG;  // 1 << (max_level + 1) and the kernels' 1 << level must stay defined
    // calcPatchSize + CV_Assert(patch.x < 6 && patch.y < 6), pyrlk.cpp:116-133,184
    const bool wide = P.win_width > 32 && P.win_width > 2 * P.win_height;
    const int bx = wide ? 32 : 16, by = wide ? 8 : 16;
    if ((P.win_width + bx - 1) / bx >= 6 || (P.win_height + by - 1) / by >= 6) return B2F_BAD_ARG;
    const size_t es = (depth == 0 ? 1 : depth == 2 ? 2 : 4) * (size_t)cn;
    if (prev_img->step < prev_img->cols * es || next_img->step < next_img->cols * es) return B2F_BAD_ARG;
    if (depth != 0 && ((prev_img->step | next_img->step) % (es / cn)) != 0) return B2F_BAD_ARG;
    if (!aligned(prev_img->data, es / cn) || !aligned(next_img->data, es / cn)) return B2F_BAD_ARG;  // element reads
    if (!aligned(prev_pts, sizeof(float2)) || !aligned(next_pts, sizeof(float2)) || !aligned(err, sizeof(float)))
        return B2F_BAD_ARG;  // the kernels read and write points as float2
    const int rows = prev_img->rows, cols = prev_img->cols;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(prev_img->data, s);
    const bool legacy = cn == 1 && (depth == 0 || depth == 5);  // single-plane texture-path kernel
    // Each point's block keeps its I, dI/dx and dI/dy patches in shared memory, 12 * cn bytes per window element.  The
    // reference holds them in registers and accepts every window calcPatchSize allows (up to 80 x 80 or 160 x 40); here
    // a patch that does not fit next to the static staging in the device's opt-in shared memory per block is refused.
    const size_t smem = sizeof(float) * 3 * (size_t)cn * P.win_width * P.win_height;
    const int optin_max = smem_optin_limit();
    if (optin_max <= 0) return B2F_CUDA_ERROR;
    if (smem + STATIC_SMEM > (size_t)optin_max) return B2F_BAD_ARG;
    const bool optin = smem + STATIC_SMEM > 48 * 1024;  // the default limit counts static and dynamic memory together

    Ctx c;
    c.stream = s;
    c.stats = &h->stats;
    if (!(h->rows == rows && h->cols == cols && h->levels == P.max_level + 1 && h->planes == cn && h->arena.capacity() > 0)) {
        if (h->arena.capacity() > 0) c.check(cudaStreamSynchronize(s));  // re-layout of a live arena
        for (int pass = 0; pass < 2 && c.ok(); ++pass) {
            Arena tmp;
            Arena &A = pass == 0 ? tmp : h->arena;
            A.begin(pass == 0);
            h->I.clear(); h->J.clear(); h->lrows.clear(); h->lcols.clear();
            int r = rows, cc = cols;
            for (int l = 0; l <= P.max_level; ++l) {
                if (l > 0) {
                    r = (r + 1) / 2;
                    cc = (cc + 1) / 2;
                }
                for (int ch = 0; ch < cn; ++ch) h->I.push_back(A.plane(r, cc));  // index l * cn + ch
                for (int ch = 0; ch < cn; ++ch) h->J.push_back(A.plane(r, cc));
                h->lrows.push_back(r);
                h->lcols.push_back(cc);
            }
            if (pass == 0) c.check(h->arena.reserve(A.used()));
        }
        if (c.ok()) {
            h->rows = rows;
            h->cols = cols;
            h->levels = P.max_level + 1;
            h->planes = cn;
        }
    }
    const int half_x = (P.win_width - 1) / 2, half_y = (P.win_height - 1) / 2;
    const float scale = static_cast<float>(1.0 / (1 << P.max_level) / 2.0);
    const float2 *init_src = reinterpret_cast<const float2 *>(P.use_initial_flow ? next_pts : prev_pts);
    if (c.ok() && legacy) {
        if (optin)
            c.check(cudaFuncSetAttribute(k_sparse_lk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const ImageView v0{prev_img->data, prev_img->step, rows, cols, prev_img->type};
        const ImageView v1{next_img->data, next_img->step, rows, cols, next_img->type};
        convert_pair(c, 1, v0, v1, h->I[0], h->J[0], 1.0f);
        const bool u8 = prev_img->type == B2F_8UC1;
        for (int l = 1; l <= P.max_level; ++l) {
            if (u8) {
                pyr_down_u8(c, 1, h->I[l - 1], h->lrows[l - 1], h->lcols[l - 1], h->I[l], h->lrows[l], h->lcols[l]);
                pyr_down_u8(c, 1, h->J[l - 1], h->lrows[l - 1], h->lcols[l - 1], h->J[l], h->lrows[l], h->lcols[l]);
            } else {
                pyr_down(c, 1, h->I[l - 1], h->lrows[l - 1], h->lcols[l - 1], h->I[l], h->lrows[l], h->lcols[l]);
                pyr_down(c, 1, h->J[l - 1], h->lrows[l - 1], h->lcols[l - 1], h->J[l], h->lrows[l], h->lcols[l]);
            }
        }
        B2F_LAUNCH(c, 2, 17.0 * n_points, k_sparse_init, dim3(div_up(n_points, 256)), dim3(256), 0, init_src,
                   reinterpret_cast<float2 *>(next_pts), status, n_points, scale);
        for (int l = P.max_level; l >= 0; --l) {
            TexView tI{h->I[l], h->lrows[l], h->lcols[l], u8 ? 0.f : 1.f};
            TexView tJ{h->J[l], h->lrows[l], h->lcols[l], u8 ? 0.f : 1.f};
            B2F_LAUNCH(c, 0, 0.0, k_sparse_lk, dim3(n_points), dim3(SB), smem, tI, tJ,
                       reinterpret_cast<const float2 *>(prev_pts), reinterpret_cast<float2 *>(next_pts), status,
                       (l == 0) ? err : nullptr, l, P.win_width, P.win_height, half_x, half_y, P.iters, u8 ? 255.0f : 1.0f);
        }
    } else if (c.ok()) {
        // sampling path per (depth, cn): the reference's sparse_caller specialisations (cuda/pyrlk.cu:575-700)
        const bool soft = cn == 3 || (depth == 2 && cn == 1) || depth == 4;
        float lo = 1.f, hi = 0.f;  // float: no rounding
        if (depth == 0) { lo = 0.f; hi = 255.f; }
        else if (depth == 2) { lo = 0.f; hi = 65535.f; }
        else if (depth == 4) { lo = -2147483648.f; hi = 2147483520.f; }
        const float norm = soft ? 1.f : (depth == 0 ? 255.f : depth == 2 ? 65535.f : 1.f);
        const float err_scale = (!soft && depth == 0) ? 255.f : 1.f;  // DenormalizationFactor<uchar>, texture path only
        auto view = [&](const std::vector<Plane> &v, int l) {
            TexViewN t{};
            for (int ch = 0; ch < cn; ++ch) t.p[ch] = v[(size_t)l * cn + ch];
            for (int ch = cn; ch < MAXC; ++ch) t.p[ch] = v[(size_t)l * cn];
            t.rows = h->lrows[l]; t.cols = h->lcols[l];
            t.norm = norm; t.lo = lo; t.hi = hi;
            return t;
        };
        {
            const dim3 block(32, 8), grid(div_up(cols, 32), div_up(rows, 8), 2);
            const double bytes = 2.0 * rows * cols * (double)(es + 4 * cn);
            TexViewN d0 = view(h->I, 0), d1 = view(h->J, 0);
            if (depth == 0)
                B2F_LAUNCH(c, 1, bytes, k_sparse_deinterleave<unsigned char>, grid, block, 0, static_cast<const unsigned char *>(prev_img->data),
                           static_cast<const unsigned char *>(next_img->data), prev_img->step, next_img->step, d0, d1, cn);
            else if (depth == 2)
                B2F_LAUNCH(c, 1, bytes, k_sparse_deinterleave<unsigned short>, grid, block, 0, static_cast<const unsigned short *>(prev_img->data),
                           static_cast<const unsigned short *>(next_img->data), prev_img->step, next_img->step, d0, d1, cn);
            else if (depth == 4)
                B2F_LAUNCH(c, 1, bytes, k_sparse_deinterleave<int>, grid, block, 0, static_cast<const int *>(prev_img->data),
                           static_cast<const int *>(next_img->data), prev_img->step, next_img->step, d0, d1, cn);
            else
                B2F_LAUNCH(c, 1, bytes, k_sparse_deinterleave<float>, grid, block, 0, static_cast<const float *>(prev_img->data),
                           static_cast<const float *>(next_img->data), prev_img->step, next_img->step, d0, d1, cn);
        }
        for (int l = 1; l <= P.max_level; ++l) {  // cuda::pyrDown on the input type: integer levels are rounded (pyr_down.cu:172)
            for (int ch = 0; ch < cn; ++ch) {
                for (int f = 0; f < 2; ++f) {
                    const std::vector<Plane> &v = f ? h->J : h->I;
                    Plane src = v[(size_t)(l - 1) * cn + ch], dst = v[(size_t)l * cn + ch];
                    pyr_down(c, 1, src, h->lrows[l - 1], h->lcols[l - 1], dst, h->lrows[l], h->lcols[l]);
                    if (depth != 5)
                        B2F_LAUNCH(c, 1, 8.0 * h->lrows[l] * h->lcols[l], k_sparse_quantize, dim3(div_up(h->lcols[l], 32), div_up(h->lrows[l], 8)),
                                   dim3(32, 8), 0, dst, h->lrows[l], h->lcols[l], lo, hi);
                }
            }
        }
        B2F_LAUNCH(c, 2, 17.0 * n_points, k_sparse_init, dim3(div_up(n_points, 256)), dim3(256), 0, init_src,
                   reinterpret_cast<float2 *>(next_pts), status, n_points, scale);
        auto launch = [&](auto kernel) {
            if (optin) c.check(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            for (int l = P.max_level; l >= 0; --l) {
                TexViewN tI = view(h->I, l), tJ = view(h->J, l);
                B2F_LAUNCH(c, 0, 0.0, kernel, dim3(n_points), dim3(SB), smem, tI, tJ, reinterpret_cast<const float2 *>(prev_pts),
                           reinterpret_cast<float2 *>(next_pts), status, (l == 0) ? err : nullptr, l, P.win_width, P.win_height,
                           half_x, half_y, P.iters, err_scale);
            }
        };
        if (cn == 1) launch(k_sparse_lk_mc<1, SAMP_SOFT>);                  // 16UC1, 32SC1
        else if (cn == 3) launch(k_sparse_lk_mc<3, SAMP_SOFT>);             // every 3-channel type
        else if (soft) launch(k_sparse_lk_mc<4, SAMP_SOFT>);                // 32SC4
        else launch(k_sparse_lk_mc<4, SAMP_TEX>);                           // 8UC4, 16UC4, 32FC4
    }
    if (c.ok() && s == nullptr) c.check(cudaDeviceSynchronize());
    if (!c.ok()) {
        h->last_cuda_error = static_cast<int>(c.err);
        cudaGetLastError();
        return c.err == cudaErrorMemoryAllocation ? B2F_OUT_OF_MEMORY : B2F_CUDA_ERROR;
    }
    return B2F_OK;
}

}  // extern "C"
