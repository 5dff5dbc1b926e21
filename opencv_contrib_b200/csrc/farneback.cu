// farneback.cu -- cv::cuda::FarnebackOpticalFlow re-implemented for sm_90a.
//
// Reference being replaced (paths relative to opencv_contrib/modules/cudaoptflow):
//   host  src/farneback.cpp:167-482   (calc / calcImpl, prepareGaussian, updateFlow_*)
//   dev   src/cuda/farneback.cu:66-595 (polynomialExpansion, updateMatrices, updateFlow,
//                                       boxFilter5, gaussianBlur, gaussianBlur5)
// plus cv::cuda::resize / pyrDown / split / merge and cv::getGaussianKernel (opencv imgproc).
//
// What is different by design (same results, fewer bytes):
//  * level images: the reference blurs the FULL-RES frame with up to 79 taps and then samples it
//    bilinearly (farneback.cpp:445-452), 12 full-frame separable blurs per pair.  Here the
//    vertical pass is evaluated only on the rows the bilinear sampling needs and the horizontal
//    pass only at the columns it needs (identical tap order and arithmetic per sample);
//  * one kernel per inner iteration: blur(M) -> updateFlow -> updateMatrices fused, the blurred M
//    never reaches HBM and the flow is only written by the level's last iteration;
//  * all tables live in the handle's arena (the reference's __constant__ tables are global state,
//    farneback.cu:60-63,154,453);
//  * one stream, no host synchronisation (the reference syncs per level, farneback.cpp:366,457).
//
// Kernel classes: 0 iter (blur5+updateFlow+updateMatrices), 1 polyexp, 2 level_image (convert,
// sparse blur, resize / pyrDown), 3 update_matrices0, 4 flow_init (prolong / split / merge).
#include "common.cuh"

#include <cuda.h>  // CUtensorMap (type only; encoded through tma_encode_2d_f32)

#include <cmath>
#include <cstring>
#include <new>
#include <vector>

namespace b2f {

namespace {

enum { CLS_ITER = 0, CLS_POLY = 1, CLS_IMG = 2, CLS_UPD0 = 3, CLS_FLOW = 4 };
constexpr int MIN_SIZE = 32;  // farneback.cpp:54
constexpr int BORDER_SIZE = 5;

// 5 planes stacked vertically in one pitched image (row k*h + y), as the reference's R / M.
struct Stack5 {
    float *p;
    int pitch, h;
    __host__ __device__ __forceinline__ float &at(int k, int y, int x) const {
        return p[((size_t)k * h + y) * pitch + x];
    }
};

struct PolyTabs {
    float g[8], xg[8], xxg[8];
    float ig11, ig03, ig33, ig55;
};

// ------------------------------------------------------------------------------------------
// host-side tables
// ------------------------------------------------------------------------------------------
// cv::getGaussianKernel(n, sigma, CV_32F) (opencv imgproc; farneback.cpp:445,462 call sites).
void gaussian_kernel(int n, double sigma, std::vector<float> &out) {
    static const double tab1[] = {1.0};
    static const double tab3[] = {0.25, 0.5, 0.25};
    static const double tab5[] = {0.0625, 0.25, 0.375, 0.25, 0.0625};
    static const double tab7[] = {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125};
    const double *fixed = nullptr;
    if (n % 2 == 1 && n <= 7 && sigma <= 0) fixed = n == 1 ? tab1 : n == 3 ? tab3 : n == 5 ? tab5 : tab7;
    const double sigmaX = sigma > 0 ? sigma : ((n - 1) * 0.5 - 1) * 0.3 + 0.8;
    const double scale2X = -0.5 / (sigmaX * sigmaX);
    std::vector<double> cf(n);
    double sum = 0;
    for (int i = 0; i < n; ++i) {
        const double x = i - (n - 1) * 0.5;
        const double t = fixed ? fixed[i] : std::exp(scale2X * x * x);
        cf[i] = t;
        sum += t;
    }
    sum = 1.0 / sum;
    out.resize(n);
    for (int i = 0; i < n; ++i) out[i] = static_cast<float>(cf[i] * sum);
}

// In-place inverse of a symmetric positive-definite 6x6 via Cholesky (DECOMP_CHOLESKY).
bool cholesky_inverse6(double A[6][6]) {
    const int n = 6;
    double L[6][6] = {};
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j <= i; ++j) {
            double s = A[i][j];
            for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
            if (i == j) {
                if (s <= 0) return false;
                L[i][i] = std::sqrt(s);
            } else {
                L[i][j] = s / L[j][j];
            }
        }
    }
    double inv[6][6];
    for (int c = 0; c < n; ++c) {
        double y[6], x[6];
        for (int i = 0; i < n; ++i) {
            double s = (i == c) ? 1.0 : 0.0;
            for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
            y[i] = s / L[i][i];
        }
        for (int i = n - 1; i >= 0; --i) {
            double s = y[i];
            for (int k = i + 1; k < n; ++k) s -= L[k][i] * x[k];
            x[i] = s / L[i][i];
        }
        for (int i = 0; i < n; ++i) inv[i][c] = x[i];
    }
    std::memcpy(A, inv, sizeof(inv));
    return true;
}

// FarnebackOpticalFlowImpl::prepareGaussian + setPolynomialExpansionConsts (farneback.cpp:209-276).
bool prepare_poly_tabs(int n, double sigma, PolyTabs &T) {
    if (sigma < FLT_EPSILON) sigma = n * 0.3;
    float gbuf[15], xgbuf[15], xxgbuf[15];
    float *g = gbuf + n, *xg = xgbuf + n, *xxg = xxgbuf + n;
    double s = 0.;
    for (int x = -n; x <= n; x++) {
        g[x] = (float)std::exp(-x * x / (2 * sigma * sigma));
        s += g[x];
    }
    s = 1. / s;
    for (int x = -n; x <= n; x++) {
        g[x] = (float)(g[x] * s);
        xg[x] = (float)(x * g[x]);
        xxg[x] = (float)(x * x * g[x]);
    }
    double G[6][6] = {};
    for (int y = -n; y <= n; y++) {
        for (int x = -n; x <= n; x++) {
            G[0][0] += g[y] * g[x];
            G[1][1] += g[y] * g[x] * x * x;
            G[3][3] += g[y] * g[x] * x * x * x * x;
            G[5][5] += g[y] * g[x] * x * x * y * y;
        }
    }
    G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
    G[4][4] = G[3][3];
    G[3][4] = G[4][3] = G[5][5];
    if (!cholesky_inverse6(G)) return false;
    std::memset(&T, 0, sizeof(T));
    for (int i = 0; i <= n; ++i) {
        T.g[i] = g[i];
        T.xg[i] = xg[i];
        T.xxg[i] = xxg[i];
    }
    T.ig11 = static_cast<float>(G[1][1]);
    T.ig03 = static_cast<float>(G[0][3]);
    T.ig33 = static_cast<float>(G[3][3]);
    T.ig55 = static_cast<float>(G[5][5]);
    return true;
}

// ------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect101(int i, int n) {
    // BrdReflect101: idx_low = |i| % n ... (single reflection is enough for |i| < 2n; loop for safety)
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        if (i >= n) i = 2 * n - 2 - i;
    }
    return i;
}

// ------------------------------------------------------------------------------------------
// level image, sparse Gaussian pre-blur (replaces gaussianBlurGpu(full frame) + cuda::resize,
// farneback.cpp:445-452; kernel arithmetic farneback.cu:455-492, resize.cu:234-269).
// V pass: Vbuf(2*y + t, x) = sum_j g[j] * (src(ry(sy - j), x) + src(ry(sy + j), x)),  sy = y1 / y2r.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_farn_blur_v(Plane f0, Plane f1, int rows, int cols, Plane v0, Plane v1,
                                                     int lrows, float inv_fy, const float *__restrict__ g,
                                                     int khalf, int identity) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int vy = blockIdx.y;  // 0 .. 2*lrows-1
    if (x >= cols) return;
    const int y = vy >> 1, t = vy & 1;
    int sy;
    if (identity) {
        if (t) return;
        sy = y;
    } else {
        const float src_y = y * inv_fy;
        const int y1 = __float2int_rd(src_y);
        if (t && (src_y - y1) == 0.f) return;  // zero bilinear weight: row never contributes
        sy = t ? min(y1 + 1, rows - 1) : min(y1, rows - 1);
    }
    const Plane src = blockIdx.z ? f1 : f0;
    float acc = __ldg(&src.at(sy, x)) * g[0];
    for (int j = 1; j <= khalf; ++j)
        acc += (__ldg(&src.at(reflect101(sy - j, rows), x)) + __ldg(&src.at(reflect101(sy + j, rows), x))) * g[j];
    (blockIdx.z ? v1 : v0).at(vy, x) = acc;
}

// Four columns per thread (the default): the kernel above gives every thread one column and a few taps -- at level 1
// of a 1080p pair 8 640 live blocks whose threads each wait out two memory round trips for three taps.  float4 loads / stores cut the blocks by four; rows whose second bilinear tap has weight
// zero for every y (integral 1 / scale, the default pyrScale = 0.5) are not launched at all (ystep = 2).  Same arithmetic
// per element: bit-identical.
__global__ void __launch_bounds__(256) k_farn_blur_v4(Plane f0, Plane f1, int rows, int cols, Plane v0, Plane v1,
                                                      int lrows, float inv_fy, const float *__restrict__ g,
                                                      int khalf, int identity, int ystep) {
    const int x = 4 * (blockIdx.x * blockDim.x + threadIdx.x);  // rows are padded to 32 floats: x + 3 stays inside the pitch
    const int vy = blockIdx.y * ystep;  // 0 .. 2*lrows-1
    if (x >= cols) return;
    const int y = vy >> 1, t = vy & 1;
    int sy;
    if (identity) {
        if (t) return;
        sy = y;
    } else {
        const float src_y = y * inv_fy;
        const int y1 = __float2int_rd(src_y);
        if (t && (src_y - y1) == 0.f) return;  // zero bilinear weight: row never contributes
        sy = t ? min(y1 + 1, rows - 1) : min(y1, rows - 1);
    }
    const Plane src = blockIdx.z ? f1 : f0;
    const float4 c = __ldg(reinterpret_cast<const float4 *>(&src.at(sy, x)));
    const float g0 = g[0];
    float4 acc = make_float4(c.x * g0, c.y * g0, c.z * g0, c.w * g0);
    for (int j = 1; j <= khalf; ++j) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(&src.at(reflect101(sy - j, rows), x)));
        const float4 b = __ldg(reinterpret_cast<const float4 *>(&src.at(reflect101(sy + j, rows), x)));
        const float gj = g[j];
        acc.x += (a.x + b.x) * gj;
        acc.y += (a.y + b.y) * gj;
        acc.z += (a.z + b.z) * gj;
        acc.w += (a.w + b.w) * gj;
    }
    *reinterpret_cast<float4 *>(&(blockIdx.z ? v1 : v0).at(vy, x)) = acc;
}

__device__ __forceinline__ float farn_hblur(const Plane &v, int vy, int sx, int cols, const float *__restrict__ g,
                                            int khalf) {
    float res = v.at(vy, sx) * g[0];
    for (int i = 1; i <= khalf; ++i)
        res += (v.at(vy, reflect101(sx - i, cols)) + v.at(vy, reflect101(sx + i, cols))) * g[i];
    return res;
}

__global__ void __launch_bounds__(256) k_farn_blur_h_resize(Plane v0, Plane v1, int rows, int cols, Plane d0, Plane d1,
                                                            int lrows, int lcols, float inv_fx, float inv_fy,
                                                            const float *__restrict__ g, int khalf, int identity) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= lcols || y >= lrows) return;
    const Plane v = blockIdx.z ? v1 : v0;
    float out;
    if (identity) {
        out = farn_hblur(v, 2 * y, x, cols, g, khalf);
    } else {
        const float src_x = x * inv_fx, src_y = y * inv_fy;
        const int x1 = __float2int_rd(src_x), y1 = __float2int_rd(src_y);
        const int x2 = x1 + 1, y2 = y1 + 1;
        const int x1r = min(x1, cols - 1), x2r = min(x2, cols - 1);
        const float wx2 = x2 - src_x, wx1 = src_x - x1;
        const float wy2 = y2 - src_y, wy1 = src_y - y1;
        out = 0.f;
        // same accumulation order as resize_linear; zero-weight taps add exactly 0 and are skipped
        out = out + farn_hblur(v, 2 * y, x1r, cols, g, khalf) * (wx2 * wy2);
        if (wx1 != 0.f) out = out + farn_hblur(v, 2 * y, x2r, cols, g, khalf) * (wx1 * wy2);
        if (wy1 != 0.f) {
            out = out + farn_hblur(v, 2 * y + 1, x1r, cols, g, khalf) * (wx2 * wy1);
            if (wx1 != 0.f) out = out + farn_hblur(v, 2 * y + 1, x2r, cols, g, khalf) * (wx1 * wy1);
        }
    }
    (blockIdx.z ? d1 : d0).at(y, x) = out;
}

// ------------------------------------------------------------------------------------------
// polynomial expansion (farneback.cu:66-119), both frames per launch.
// Block = 32 x 8 output pixels.  Vertical pass for the 32+2n columns of the block into shared
// memory (3 moments), then the horizontal pass; replicate clamping as the reference.
// ------------------------------------------------------------------------------------------
template <int N>
__global__ void __launch_bounds__(256) k_farn_polyexp(Plane s0, Plane s1, Stack5 r0, Stack5 r1, int rows, int cols,
                                                      PolyTabs T) {
    constexpr int TW = 32, TH = 8, SW = TW + 2 * N;
    __shared__ float sm[3][TH][SW];
    const Plane src = blockIdx.z ? s1 : s0;
    const Stack5 dst = blockIdx.z ? r1 : r0;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int x0 = blockIdx.x * TW, y = blockIdx.y * TH + ty;
    if (y < rows) {
        for (int i = tx; i < SW; i += TW) {
            const int xc = clampi(x0 + i - N, 0, cols - 1);
            float a0 = __ldg(&src.at(y, xc)) * T.g[0], a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int k = 1; k <= N; ++k) {
                const float t0 = __ldg(&src.at(max(y - k, 0), xc));
                const float t1 = __ldg(&src.at(min(y + k, rows - 1), xc));
                a0 += T.g[k] * (t0 + t1);
                a1 += T.xg[k] * (t1 - t0);
                a2 += T.xxg[k] * (t0 + t1);
            }
            sm[0][ty][i] = a0;
            sm[1][ty][i] = a1;
            sm[2][ty][i] = a2;
        }
    }
    __syncthreads();
    const int x = x0 + tx;
    if (y >= rows || x >= cols) return;
    const float *row0 = &sm[0][ty][tx + N], *row1 = &sm[1][ty][tx + N], *row2 = &sm[2][ty][tx + N];
    float b1 = T.g[0] * row0[0], b3 = T.g[0] * row1[0], b5 = T.g[0] * row2[0];
    float b2 = 0.f, b4 = 0.f, b6 = 0.f;
#pragma unroll
    for (int k = 1; k <= N; ++k) {
        b1 += (row0[k] + row0[-k]) * T.g[k];
        b4 += (row0[k] + row0[-k]) * T.xxg[k];
        b2 += (row0[k] - row0[-k]) * T.xg[k];
        b3 += (row1[k] + row1[-k]) * T.g[k];
        b6 += (row1[k] - row1[-k]) * T.xg[k];
        b5 += (row2[k] + row2[-k]) * T.g[k];
    }
    dst.at(0, y, x) = b3 * T.ig11;
    dst.at(1, y, x) = b2 * T.ig11;
    dst.at(2, y, x) = b1 * T.ig03 + b5 * T.ig33;
    dst.at(3, y, x) = b1 * T.ig03 + b4 * T.ig33;
    dst.at(4, y, x) = b6 * T.ig55;
}

// Register-blocked variant (the default): in the kernel above every output of the vertical pass issues its own 2N+1
// loads, the second round of its 32-lane column loop is two thirds empty (42 columns), and the horizontal pass reads
// 6N+3 scalars from shared memory per pixel.  Here one block = 64 x 32 pixels; a vertical task is (column, 8-row segment): 8+2N loads feed 8 outputs
// from a register window; a horizontal task is (row, 4 pixels): 4 (N = 5) or 5 (N = 7) LDS.128 per moment feed 4 outputs, and
// the five results leave as float4.  Same expressions in the same order per output: bit-identical (tested; aux_path 6 keeps
// the kernel above).
template <int N>
__global__ void __launch_bounds__(256) k_farn_polyexp_fast(Plane s0, Plane s1, Stack5 r0, Stack5 r1, int rows, int cols,
                                                           PolyTabs T) {
    constexpr int TW = 64, TH = 32, NC = TW + 2 * N, SW = (NC + 3) & ~3, SEG = 8, WIN = SEG + 2 * N;
    constexpr int HW = 4 + 2 * N, HV = (HW + 3) / 4;  // horizontal window (floats / float4s)
    __shared__ __align__(16) float sm[3][TH][SW];
    const Plane src = blockIdx.z ? s1 : s0;
    const Stack5 dst = blockIdx.z ? r1 : r0;
    const int tid = threadIdx.y * 32 + threadIdx.x;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;

    for (int task = tid; task < NC * (TH / SEG); task += 256) {
        const int seg = task / NC, i = task - seg * NC;
        const int ys = y0 + seg * SEG;
        if (ys >= rows) continue;
        const int xc = clampi(x0 + i - N, 0, cols - 1);
        float v[WIN];
        if (ys - N >= 0 && ys - N + WIN <= rows) {
            const float *p = &src.at(ys - N, xc);
#pragma unroll
            for (int q = 0; q < WIN; ++q) {
                v[q] = __ldg(p);
                p += src.pitch;
            }
        } else {
#pragma unroll
            for (int q = 0; q < WIN; ++q) v[q] = __ldg(&src.at(clampi(ys - N + q, 0, rows - 1), xc));
        }
#pragma unroll
        for (int o = 0; o < SEG; ++o) {
            float a0 = v[o + N] * T.g[0], a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int k = 1; k <= N; ++k) {
                const float t0 = v[o + N - k];
                const float t1 = v[o + N + k];
                a0 += T.g[k] * (t0 + t1);
                a1 += T.xg[k] * (t1 - t0);
                a2 += T.xxg[k] * (t0 + t1);
            }
            sm[0][seg * SEG + o][i] = a0;
            sm[1][seg * SEG + o][i] = a1;
            sm[2][seg * SEG + o][i] = a2;
        }
    }
    __syncthreads();

    for (int task = tid; task < TH * (TW / 4); task += 256) {
        const int r = task / (TW / 4), q = task - r * (TW / 4);
        const int y = y0 + r, x = x0 + 4 * q;
        if (y >= rows || x >= cols) continue;
        float w0[4 * HV], w1[4 * HV], w2[4 * HV];  // window columns 4q .. 4q + 4 HV - 1 (centre of pixel e at e + N)
#pragma unroll
        for (int c = 0; c < HV; ++c) {
            const float4 a = *reinterpret_cast<const float4 *>(&sm[0][r][4 * q + 4 * c]);
            const float4 b = *reinterpret_cast<const float4 *>(&sm[1][r][4 * q + 4 * c]);
            const float4 d = *reinterpret_cast<const float4 *>(&sm[2][r][4 * q + 4 * c]);
            w0[4 * c] = a.x; w0[4 * c + 1] = a.y; w0[4 * c + 2] = a.z; w0[4 * c + 3] = a.w;
            w1[4 * c] = b.x; w1[4 * c + 1] = b.y; w1[4 * c + 2] = b.z; w1[4 * c + 3] = b.w;
            w2[4 * c] = d.x; w2[4 * c + 1] = d.y; w2[4 * c + 2] = d.z; w2[4 * c + 3] = d.w;
        }
        float o0[4], o1[4], o2[4], o3[4], o4[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int c = e + N;
            float b1 = T.g[0] * w0[c], b3 = T.g[0] * w1[c], b5 = T.g[0] * w2[c];
            float b2 = 0.f, b4 = 0.f, b6 = 0.f;
#pragma unroll
            for (int k = 1; k <= N; ++k) {
                b1 += (w0[c + k] + w0[c - k]) * T.g[k];
                b4 += (w0[c + k] + w0[c - k]) * T.xxg[k];
                b2 += (w0[c + k] - w0[c - k]) * T.xg[k];
                b3 += (w1[c + k] + w1[c - k]) * T.g[k];
                b6 += (w1[c + k] - w1[c - k]) * T.xg[k];
                b5 += (w2[c + k] + w2[c - k]) * T.g[k];
            }
            o0[e] = b3 * T.ig11;
            o1[e] = b2 * T.ig11;
            o2[e] = b1 * T.ig03 + b5 * T.ig33;
            o3[e] = b1 * T.ig03 + b4 * T.ig33;
            o4[e] = b6 * T.ig55;
        }
        if (x + 3 < cols) {
            *reinterpret_cast<float4 *>(&dst.at(0, y, x)) = make_float4(o0[0], o0[1], o0[2], o0[3]);
            *reinterpret_cast<float4 *>(&dst.at(1, y, x)) = make_float4(o1[0], o1[1], o1[2], o1[3]);
            *reinterpret_cast<float4 *>(&dst.at(2, y, x)) = make_float4(o2[0], o2[1], o2[2], o2[3]);
            *reinterpret_cast<float4 *>(&dst.at(3, y, x)) = make_float4(o3[0], o3[1], o3[2], o3[3]);
            *reinterpret_cast<float4 *>(&dst.at(4, y, x)) = make_float4(o4[0], o4[1], o4[2], o4[3]);
        } else {
            for (int e = 0; e < 4 && x + e < cols; ++e) {
                dst.at(0, y, x + e) = o0[e];
                dst.at(1, y, x + e) = o1[e];
                dst.at(2, y, x + e) = o2[e];
                dst.at(3, y, x + e) = o3[e];
                dst.at(4, y, x + e) = o4[e];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// updateMatrices for one pixel (farneback.cu:156-241).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float farn_border_w(int d) {
    // c_border = {0.14, 0.14, 0.4472, 0.4472, 0.4472, 1} (farneback.cu:246)
    return d <= 1 ? 0.14f : (d < BORDER_SIZE ? 0.4472f : 1.f);
}

__device__ __forceinline__ void farn_update_matrices_px(const Stack5 &R0, const Stack5 &R1, int rows, int cols, int x,
                                                        int y, float dx, float dy, float (&m)[5]) {
    float fx = x + dx, fy = y + dy;
    // floorf of a wild flow must not overflow the int conversion
    const float ffx = fminf(fmaxf(floorf(fx), -4.f), (float)cols + 4.f);
    const float ffy = fminf(fmaxf(floorf(fy), -4.f), (float)rows + 4.f);
    const int x1 = (int)ffx, y1 = (int)ffy;
    fx -= floorf(fx);
    fy -= floorf(fy);
    float r2, r3, r4, r5, r6;
    if (x1 >= 0 && y1 >= 0 && x1 < cols - 1 && y1 < rows - 1) {
        const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy);
        const float a10 = (1.f - fx) * fy, a11 = fx * fy;
        const float *p = &R1.at(0, y1, x1);
        const size_t ps = (size_t)R1.h * R1.pitch;
        const int pitch = R1.pitch;
        r2 = a00 * __ldg(p) + a01 * __ldg(p + 1) + a10 * __ldg(p + pitch) + a11 * __ldg(p + pitch + 1);
        p += ps;
        r3 = a00 * __ldg(p) + a01 * __ldg(p + 1) + a10 * __ldg(p + pitch) + a11 * __ldg(p + pitch + 1);
        p += ps;
        r4 = a00 * __ldg(p) + a01 * __ldg(p + 1) + a10 * __ldg(p + pitch) + a11 * __ldg(p + pitch + 1);
        p += ps;
        r5 = a00 * __ldg(p) + a01 * __ldg(p + 1) + a10 * __ldg(p + pitch) + a11 * __ldg(p + pitch + 1);
        p += ps;
        r6 = a00 * __ldg(p) + a01 * __ldg(p + 1) + a10 * __ldg(p + pitch) + a11 * __ldg(p + pitch + 1);
        r4 = (__ldg(&R0.at(2, y, x)) + r4) * 0.5f;
        r5 = (__ldg(&R0.at(3, y, x)) + r5) * 0.5f;
        r6 = (__ldg(&R0.at(4, y, x)) + r6) * 0.25f;
    } else {
        r2 = r3 = 0.f;
        r4 = __ldg(&R0.at(2, y, x));
        r5 = __ldg(&R0.at(3, y, x));
        r6 = __ldg(&R0.at(4, y, x)) * 0.5f;
    }
    r2 = (__ldg(&R0.at(0, y, x)) - r2) * 0.5f;
    r3 = (__ldg(&R0.at(1, y, x)) - r3) * 0.5f;
    r2 += r4 * dy + r6 * dx;
    r3 += r6 * dy + r5 * dx;
    const float scale = farn_border_w(min(x, BORDER_SIZE)) * farn_border_w(min(y, BORDER_SIZE)) *
                        farn_border_w(min(cols - x - 1, BORDER_SIZE)) * farn_border_w(min(rows - y - 1, BORDER_SIZE));
    r2 *= scale; r3 *= scale; r4 *= scale; r5 *= scale; r6 *= scale;
    m[0] = r4 * r4 + r6 * r6;
    m[1] = (r4 + r5) * r6;
    m[2] = r5 * r5 + r6 * r6;
    m[3] = r4 * r2 + r6 * r3;
    m[4] = r6 * r2 + r5 * r3;
}


// updateMatrices for 4 horizontally adjacent pixels (x multiple of 4), arranged plane-major so that the
// 16 bilinear-gather loads of one R1 plane are all in flight together (the per-pixel form exposes one
// L2 round trip per pixel).  Same arithmetic per pixel as farn_update_matrices_px.
__device__ __forceinline__ void farn_update_matrices_quad(const Stack5 &R0, const Stack5 &R1, int rows, int cols,
                                                          int x, int y, const float (&dx)[4], const float (&dy)[4],
                                                          float (&m)[4][5]) {
    float a00[4], a01[4], a10[4], a11[4];
    const float *base[4];
    bool inb[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float fx = (x + e) + dx[e], fy = y + dy[e];
        const float ffx = fminf(fmaxf(floorf(fx), -4.f), (float)cols + 4.f);
        const float ffy = fminf(fmaxf(floorf(fy), -4.f), (float)rows + 4.f);
        const int x1 = (int)ffx, y1 = (int)ffy;
        fx -= floorf(fx);
        fy -= floorf(fy);
        inb[e] = x1 >= 0 && y1 >= 0 && x1 < cols - 1 && y1 < rows - 1 && x + e < cols;
        a00[e] = (1.f - fx) * (1.f - fy);
        a01[e] = fx * (1.f - fy);
        a10[e] = (1.f - fx) * fy;
        a11[e] = fx * fy;
        base[e] = &R1.at(0, inb[e] ? y1 : 0, inb[e] ? x1 : 0);
    }
    const size_t ps = (size_t)R1.h * R1.pitch;
    const int pitch = R1.pitch;
    float g[5][4];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        float t00[4], t01[4], t10[4], t11[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float *p = base[e];
            const float *p2 = p + pitch;
            t00[e] = __ldg(p);
            t01[e] = __ldg(p + 1);
            t10[e] = __ldg(p2);
            t11[e] = __ldg(p2 + 1);
            base[e] = p + ps;  // next plane
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) g[k][e] = a00[e] * t00[e] + a01[e] * t01[e] + a10[e] * t10[e] + a11[e] * t11[e];
    }
    float r0v[5][4];
    const bool full = x + 3 < cols;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        if (full) {
            const float4 t = __ldg(reinterpret_cast<const float4 *>(&R0.at(k, y, x)));
            r0v[k][0] = t.x; r0v[k][1] = t.y; r0v[k][2] = t.z; r0v[k][3] = t.w;
        } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) r0v[k][e] = x + e < cols ? __ldg(&R0.at(k, y, x + e)) : 0.f;
        }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float r2, r3, r4, r5, r6;
        if (inb[e]) {
            r2 = g[0][e];
            r3 = g[1][e];
            r4 = (r0v[2][e] + g[2][e]) * 0.5f;
            r5 = (r0v[3][e] + g[3][e]) * 0.5f;
            r6 = (r0v[4][e] + g[4][e]) * 0.25f;
        } else {
            r2 = r3 = 0.f;
            r4 = r0v[2][e];
            r5 = r0v[3][e];
            r6 = r0v[4][e] * 0.5f;
        }
        r2 = (r0v[0][e] - r2) * 0.5f;
        r3 = (r0v[1][e] - r3) * 0.5f;
        r2 += r4 * dy[e] + r6 * dx[e];
        r3 += r6 * dy[e] + r5 * dx[e];
        const int xe = x + e;
        const float scale = farn_border_w(min(xe, BORDER_SIZE)) * farn_border_w(min(y, BORDER_SIZE)) *
                            farn_border_w(min(cols - xe - 1, BORDER_SIZE)) * farn_border_w(min(rows - y - 1, BORDER_SIZE));
        r2 *= scale; r3 *= scale; r4 *= scale; r5 *= scale; r6 *= scale;
        m[e][0] = r4 * r4 + r6 * r6;
        m[e][1] = (r4 + r5) * r6;
        m[e][2] = r5 * r5 + r6 * r6;
        m[e][3] = r4 * r2 + r6 * r3;
        m[e][4] = r6 * r2 + r5 * r3;
    }
}


// updateMatrices for 4 pixels at arbitrary positions (xs[e], ys[e]); used by the lane-transposed gather of
// k_farn_iter_fast, where lane L of a warp owns pixels L, L+32 of two tile rows: one gather instruction of the warp
// then covers 32 CONSECUTIVE pixels (4-6 sectors) instead of every fourth pixel of 128 (16 sectors, a quarter of each
// used).  Same arithmetic per pixel as farn_update_matrices_px / _quad; ok[e] = pixel inside the image.
__device__ __forceinline__ void farn_update_matrices_spread(const Stack5 &R0, const Stack5 &R1, int rows, int cols,
                                                            const int (&xs)[4], const int (&ys)[4], const bool (&ok)[4],
                                                            const float (&dx)[4], const float (&dy)[4],
                                                            float (&m)[4][5]) {
    float a00[4], a01[4], a10[4], a11[4];
    const float *base[4];
    bool inb[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float fx = xs[e] + dx[e], fy = ys[e] + dy[e];
        const float ffx = fminf(fmaxf(floorf(fx), -4.f), (float)cols + 4.f);
        const float ffy = fminf(fmaxf(floorf(fy), -4.f), (float)rows + 4.f);
        const int x1 = (int)ffx, y1 = (int)ffy;
        fx -= floorf(fx);
        fy -= floorf(fy);
        inb[e] = x1 >= 0 && y1 >= 0 && x1 < cols - 1 && y1 < rows - 1 && ok[e];
        a00[e] = (1.f - fx) * (1.f - fy);
        a01[e] = fx * (1.f - fy);
        a10[e] = (1.f - fx) * fy;
        a11[e] = fx * fy;
        base[e] = &R1.at(0, inb[e] ? y1 : 0, inb[e] ? x1 : 0);
    }
    const size_t ps = (size_t)R1.h * R1.pitch;
    const int pitch = R1.pitch;
    float g[5][4];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        float t00[4], t01[4], t10[4], t11[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float *p = base[e];
            const float *p2 = p + pitch;
            t00[e] = __ldg(p);
            t01[e] = __ldg(p + 1);
            t10[e] = __ldg(p2);
            t11[e] = __ldg(p2 + 1);
            base[e] = p + ps;  // next plane
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) g[k][e] = a00[e] * t00[e] + a01[e] * t01[e] + a10[e] * t10[e] + a11[e] * t11[e];
    }
    float r0v[5][4];
#pragma unroll
    for (int k = 0; k < 5; ++k)
#pragma unroll
        for (int e = 0; e < 4; ++e) r0v[k][e] = ok[e] ? __ldg(&R0.at(k, ys[e], xs[e])) : 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float r2, r3, r4, r5, r6;
        if (inb[e]) {
            r2 = g[0][e];
            r3 = g[1][e];
            r4 = (r0v[2][e] + g[2][e]) * 0.5f;
            r5 = (r0v[3][e] + g[3][e]) * 0.5f;
            r6 = (r0v[4][e] + g[4][e]) * 0.25f;
        } else {
            r2 = r3 = 0.f;
            r4 = r0v[2][e];
            r5 = r0v[3][e];
            r6 = r0v[4][e] * 0.5f;
        }
        r2 = (r0v[0][e] - r2) * 0.5f;
        r3 = (r0v[1][e] - r3) * 0.5f;
        r2 += r4 * dy[e] + r6 * dx[e];
        r3 += r6 * dy[e] + r5 * dx[e];
        const int xe = xs[e], ye = ys[e];
        const float scale = farn_border_w(min(xe, BORDER_SIZE)) * farn_border_w(min(ye, BORDER_SIZE)) *
                            farn_border_w(min(cols - xe - 1, BORDER_SIZE)) * farn_border_w(min(rows - ye - 1, BORDER_SIZE));
        r2 *= scale; r3 *= scale; r4 *= scale; r5 *= scale; r6 *= scale;
        m[e][0] = r4 * r4 + r6 * r6;
        m[e][1] = (r4 + r5) * r6;
        m[e][2] = r5 * r5 + r6 * r6;
        m[e][3] = r4 * r2 + r6 * r3;
        m[e][4] = r6 * r2 + r5 * r3;
    }
}

__global__ void __launch_bounds__(256) k_farn_update_matrices(Plane flowx, Plane flowy, Stack5 R0, Stack5 R1, Stack5 M,
                                                              int rows, int cols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    float m[5];
    farn_update_matrices_px(R0, R1, rows, cols, x, y, flowx.at(y, x), flowy.at(y, x), m);
#pragma unroll
    for (int k = 0; k < 5; ++k) M.at(k, y, x) = m[k];
}

// ------------------------------------------------------------------------------------------
// fused inner iteration: blur5(M) -> updateFlow -> updateMatrices
// (boxFilter5 farneback.cu:357-412 / gaussianBlur5 :539-595, updateFlow :267-286, updateMatrices).
// Block = 64 x 8 output pixels, 256 threads (each thread: 2 pixels in x).  The vertical pass is
// computed for the 64 + 2k columns of the block straight from M (L1/L2 hits, replicate clamp) into
// shared memory; the horizontal pass, the 2x2 solve and the matrix update run from there.
// GAUSS = false: plain sums then * 1/area.  GAUSS = true: taps g[] (replicate border).
// ------------------------------------------------------------------------------------------
constexpr int IT_TW = 64, IT_TH = 8;

template <bool GAUSS>
__global__ void __launch_bounds__(256) k_farn_iter(Stack5 Min, Stack5 Mout, Stack5 R0, Stack5 R1, Plane flowx,
                                                   Plane flowy, int rows, int cols, int khalf, float box_inv,
                                                   const float *__restrict__ g, int update_matrices,
                                                   int write_flow) {
    extern __shared__ float sm[];  // [5][IT_TH][sw]
    const int sw = IT_TW + 2 * khalf;
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * IT_TW, y0 = blockIdx.y * IT_TH;

    // vertical pass: (column i, row r) pairs spread over the block
    for (int idx = tid; idx < sw * IT_TH; idx += 256) {
        const int r = idx / sw, i = idx - r * sw;
        const int y = y0 + r;
        if (y >= rows) continue;
        const int xc = clampi(x0 + i - khalf, 0, cols - 1);
        float acc[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const float c = __ldg(&Min.at(k, y, xc));
            acc[k] = GAUSS ? c * g[0] : c;
        }
        for (int j = 1; j <= khalf; ++j) {
            const int ya = max(y - j, 0), yb = min(y + j, rows - 1);
            const float gj = GAUSS ? g[j] : 1.f;
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const float s = __ldg(&Min.at(k, ya, xc)) + __ldg(&Min.at(k, yb, xc));
                acc[k] = GAUSS ? acc[k] + s * gj : acc[k] + s;
            }
        }
#pragma unroll
        for (int k = 0; k < 5; ++k) sm[(k * IT_TH + r) * sw + i] = acc[k];
    }
    __syncthreads();

    const int r = tid >> 5;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int lx = (tid & 31) + 32 * half;
        const int x = x0 + lx, y = y0 + r;
        if (x >= cols || y >= rows) continue;
        float res[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const float *row = &sm[(k * IT_TH + r) * sw + lx + khalf];
            float a = GAUSS ? row[0] * g[0] : row[0];
            for (int i = 1; i <= khalf; ++i) a = GAUSS ? a + (row[-i] + row[i]) * g[i] : a + (row[-i] + row[i]);
            res[k] = GAUSS ? a : a * box_inv;
        }
        // updateFlow
        const float g11 = res[0], g12 = res[1], g22 = res[2], h1 = res[3], h2 = res[4];
        const float detInv = 1.f / (g11 * g22 - g12 * g12 + 1e-3f);
        const float fx = (g11 * h2 - g12 * h1) * detInv;
        const float fy = (g22 * h1 - g12 * h2) * detInv;
        if (write_flow) {
            flowx.at(y, x) = fx;
            flowy.at(y, x) = fy;
        }
        if (update_matrices) {
            float m[5];
            farn_update_matrices_px(R0, R1, rows, cols, x, y, fx, fy, m);
#pragma unroll
            for (int k = 0; k < 5; ++k) Mout.at(k, y, x) = m[k];
        }
    }
}


// ------------------------------------------------------------------------------------------
// Register-blocked variant of the fused iteration for a compile-time window half-size K
// (winSize = 2K+1; K = 6 is the reference default 13).  Same arithmetic and summation order as
// k_farn_iter, ~4x fewer instructions:
//   vertical pass   one task = (column, plane, 16-row half): 16+2K loads feed 16 outputs from a
//                   register window instead of 2K+1 loads per output;
//   horizontal pass one task = (row, 4 consecutive pixels): 4 LDS.128 per plane feed 4 outputs;
//   R0 / M / flow   move as float4.
// Block = 64 x 32 output pixels, 256 threads, 5*32*(64+2K)*4 B shared memory.
// ------------------------------------------------------------------------------------------
// sum of the first N elements as a balanced tree (short dependency chain)
template <int N, int M>
__device__ __forceinline__ float box_first(const float (&v)[M]) {
    static_assert(N == 13 && M >= N, "window of 13");
    const float a = (v[0] + v[1]) + (v[2] + v[3]), b = (v[4] + v[5]) + (v[6] + v[7]);
    const float c = (v[8] + v[9]) + (v[10] + v[11]);
    return ((a + b) + c) + v[12];
}

constexpr int FT_W = 64, FT_H = 32;

template <int K, bool GAUSS, bool QUAD, int NT = 256, int MINB = (NT == 256 ? 2 : 1), bool XPOSE = false>
__global__ void __launch_bounds__(NT, MINB) k_farn_iter_fast(Stack5 Min, Stack5 Mout, Stack5 R0, Stack5 R1, Plane flowx,
                                                        Plane flowy, int rows, int cols, float box_inv,
                                                        const float *__restrict__ g, int update_matrices,
                                                        int write_flow) {
    constexpr int SW = FT_W + 2 * K;  // staged columns (multiple of 4 for even K)
    constexpr int HALF = FT_H / 2;
    constexpr int WIN = HALF + 2 * K;
    extern __shared__ __align__(16) float sm[];  // [5][FT_H][SW]
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * FT_W, y0 = blockIdx.y * FT_H;

    float gk[K + 1];
#pragma unroll
    for (int j = 0; j <= K; ++j) gk[j] = GAUSS ? g[j] : 1.f;

    // ---- vertical pass ----
    const size_t plane_stride = (size_t)Min.h * Min.pitch;
    for (int task = tid; task < SW * 5 * 2; task += NT) {
        const int half = task / (SW * 5);
        const int rem = task - half * (SW * 5);
        const int pl = rem / SW, i = rem - pl * SW;
        const int xc = clampi(x0 + i - K, 0, cols - 1);
        const int yb = y0 + half * HALF - K;
        const float *colp = Min.p + pl * plane_stride + xc;  // column base of this plane
        float v[WIN];
        if (yb >= 0 && yb + WIN <= rows) {  // interior rows: walk the column with one pointer
            const float *p = colp + (size_t)yb * Min.pitch;
#pragma unroll
            for (int q = 0; q < WIN; ++q) {
                v[q] = __ldg(p);
                p += Min.pitch;
            }
        } else {
#pragma unroll
            for (int q = 0; q < WIN; ++q) v[q] = __ldg(colp + (size_t)clampi(yb + q, 0, rows - 1) * Min.pitch);
        }
        float *dst = sm + ((size_t)pl * FT_H + half * HALF) * SW + i;
        if (GAUSS) {
#pragma unroll
            for (int o = 0; o < HALF; ++o) {
                float acc = v[o + K] * gk[0];
#pragma unroll
                for (int j = 1; j <= K; ++j) acc = acc + (v[o + K - j] + v[o + K + j]) * gk[j];
                dst[o * SW] = acc;
            }
        } else {
            // box window: running sum (one window of 2K+1 adds, then +new -old per output) instead of 2K adds per
            // output -- 44 instead of 192 additions for 16 outputs; the CPU reference slides its vertical sums too
            float acc = box_first<2 * K + 1>(v);
            dst[0] = acc;
#pragma unroll
            for (int o = 1; o < HALF; ++o) {
                acc = acc + (v[o + 2 * K] - v[o - 1]);
                dst[o * SW] = acc;
            }
        }
    }
    __syncthreads();

    // ---- horizontal pass + 2x2 solve + matrix update, 4 pixels per task ----
#pragma unroll 1
    for (int task = tid; task < FT_H * (FT_W / 4); task += NT) {
        const int r = task / (FT_W / 4), q = task - r * (FT_W / 4);
        const int y = y0 + r, x = x0 + 4 * q;
        const bool live = y < rows && x < cols;
        if (!XPOSE && !live) continue;  // the transposed gather below needs the whole warp
        float res[5][4];
#pragma unroll
        for (int pl = 0; pl < 5; ++pl) {
            const float *row = sm + ((size_t)pl * FT_H + r) * SW + 4 * q;
            float w[4 + 2 * K + 2];
#pragma unroll
            for (int c = 0; c < (4 + 2 * K + 3) / 4; ++c) {
                const float4 t = *reinterpret_cast<const float4 *>(row + 4 * c);
                w[4 * c] = t.x;
                w[4 * c + 1] = t.y;
                if (4 * c + 2 < 4 + 2 * K + 2) w[4 * c + 2] = t.z;
                if (4 * c + 3 < 4 + 2 * K + 2) w[4 * c + 3] = t.w;
            }
            if (GAUSS) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float acc = w[e + K] * gk[0];
#pragma unroll
                    for (int i = 1; i <= K; ++i) acc = acc + (w[e + K - i] + w[e + K + i]) * gk[i];
                    res[pl][e] = acc;
                }
            } else {
                float acc = box_first<2 * K + 1>(w);
                res[pl][0] = acc * box_inv;
#pragma unroll
                for (int e = 1; e < 4; ++e) {
                    acc = acc + (w[e + 2 * K] - w[e - 1]);
                    res[pl][e] = acc * box_inv;
                }
            }
        }
        float fx[4], fy[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float g11 = res[0][e], g12 = res[1][e], g22 = res[2][e], h1 = res[3][e], h2 = res[4][e];
            const float detInv = 1.f / (g11 * g22 - g12 * g12 + 1e-3f);
            fx[e] = (g11 * h2 - g12 * h1) * detInv;
            fy[e] = (g22 * h1 - g12 * h2) * detInv;
        }
        const bool full = x + 3 < cols;
        if (write_flow && live) {
            if (full) {
                *reinterpret_cast<float4 *>(&flowx.at(y, x)) = make_float4(fx[0], fx[1], fx[2], fx[3]);
                *reinterpret_cast<float4 *>(&flowy.at(y, x)) = make_float4(fy[0], fy[1], fy[2], fy[3]);
            } else {
                for (int e = 0; e < 4 && x + e < cols; ++e) {
                    flowx.at(y, x + e) = fx[e];
                    flowy.at(y, x + e) = fy[e];
                }
            }
        }
        if (XPOSE && update_matrices) {
            // hand the displacements over to the lane-transposed mapping: the warp's two tile rows (2 x 64 pixels) go
            // through a 1 KB buffer; lane L then owns columns L and L + 32 of both rows
            const int lane = tid & 31;
            float *tb = sm + 5 * FT_H * SW + (tid >> 5) * 256;  // [fx | fy][2 rows][64]
            __syncwarp();
            *reinterpret_cast<float4 *>(tb + (lane >> 4) * FT_W + 4 * (lane & 15)) = make_float4(fx[0], fx[1], fx[2], fx[3]);
            *reinterpret_cast<float4 *>(tb + 128 + (lane >> 4) * FT_W + 4 * (lane & 15)) = make_float4(fy[0], fy[1], fy[2], fy[3]);
            __syncwarp();
            const int rw = (task - lane) / (FT_W / 4);  // first of the warp's two rows
            int xs[4], ys[4];
            bool ok[4];
            float dxs[4], dys[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int rr = e >> 1, cc = lane + 32 * (e & 1);
                xs[e] = x0 + cc;
                ys[e] = y0 + rw + rr;
                ok[e] = xs[e] < cols && ys[e] < rows;
                dxs[e] = tb[rr * FT_W + cc];
                dys[e] = tb[128 + rr * FT_W + cc];
            }
            float m[4][5];
            farn_update_matrices_spread(R0, R1, rows, cols, xs, ys, ok, dxs, dys, m);
#pragma unroll
            for (int pl = 0; pl < 5; ++pl)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (ok[e]) Mout.at(pl, ys[e], xs[e]) = m[e][pl];
        } else if (update_matrices) {
            float m[4][5];
            if (QUAD) {
                farn_update_matrices_quad(R0, R1, rows, cols, x, y, fx, fy, m);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (x + e < cols) farn_update_matrices_px(R0, R1, rows, cols, x + e, y, fx[e], fy[e], m[e]);
                    else { m[e][0] = m[e][1] = m[e][2] = m[e][3] = m[e][4] = 0.f; }
                }
            }
#pragma unroll
            for (int pl = 0; pl < 5; ++pl) {
                if (full) {
                    *reinterpret_cast<float4 *>(&Mout.at(pl, y, x)) = make_float4(m[0][pl], m[1][pl], m[2][pl], m[3][pl]);
                } else {
                    for (int e = 0; e < 4 && x + e < cols; ++e) Mout.at(pl, y, x + e) = m[e][pl];
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host engine
// ------------------------------------------------------------------------------------------
// Persistent TMA variant of the fast kernel for levels with many tiles (opt-in: kernel_path = 3).
// One 512-thread CTA per SM walks 64x64 tiles.  The five M planes of a tile (+6 halo, rounded out to a 16-byte
// aligned 80-column box) arrive through cp.async.bulk.tensor into shared memory, so the vertical pass reads
// shared memory instead of issuing three dependent rounds of global loads per thread; as soon as the vertical
// sums are formed the NEXT tile's boxes are requested into the same buffer and land while this tile runs its
// horizontal pass, solve and R1 gather.  TMA zero-fills outside the tensor, the blur needs replicate borders:
// border tiles patch their halo cells from the clamped in-tile position before the vertical pass.
// Same arithmetic and summation order as k_farn_iter_fast -> bit-identical.
// ------------------------------------------------------------------------------------------
constexpr int TT = 64;              // tile edge
constexpr int TB_W = TT + 16;       // box columns: x0-8 .. x0+71 (origin a multiple of 4 floats)
constexpr int TB_H = TT + 12;       // box rows:    y0-6 .. y0+69
constexpr int TSW = TT + 12;        // vertical-sum columns: x0-6 .. x0+69
constexpr int TNT = 512;
constexpr size_t FARN_TMA_SMEM = sizeof(float) * (5 * TB_H * TB_W + 5 * TT * TSW) + 64;

__device__ __forceinline__ uint32_t farn_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void farn_mbar_wait(uint64_t *bar, uint32_t parity) {
    // bounded: a descriptor / byte-count mistake must trap, not hang the GPU
    for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
        uint32_t ok;
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}" : "=r"(ok) : "r"(farn_smem_u32(bar)), "r"(parity) : "memory");
        if (ok) return;
    }
    __trap();
}

template <bool GAUSS>
__global__ void __launch_bounds__(TNT, 1)
    k_farn_iter_tma(const __grid_constant__ CUtensorMap mapM, Stack5 Mout, Stack5 R0, Stack5 R1, Plane flowx, Plane flowy,
                    int rows, int cols, int plane_rows, float box_inv, const float *__restrict__ g, int update_matrices,
                    int write_flow, int tiles_x, int ntiles) {
    constexpr int K = 6;
    extern __shared__ __align__(1024) float tsm[];
    float *inbuf = tsm;                      // [5][TB_H][TB_W]
    float *sums = tsm + 5 * TB_H * TB_W;     // [5][TT][TSW]
    uint64_t *bar = reinterpret_cast<uint64_t *>(sums + 5 * TT * TSW);
    const int tid = threadIdx.x;
    constexpr uint32_t kBytes = 5 * TB_H * TB_W * sizeof(float);

    float gk[K + 1];
#pragma unroll
    for (int j = 0; j <= K; ++j) gk[j] = GAUSS ? g[j] : 1.f;

    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(farn_smem_u32(bar)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    auto request = [&](int t) {  // thread 0 only
        const int ty = t / tiles_x, tx = t - ty * tiles_x;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(farn_smem_u32(bar)), "r"(kBytes) : "memory");
#pragma unroll
        for (int pl = 0; pl < 5; ++pl)
            asm volatile(
                "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                ::"r"(farn_smem_u32(inbuf + pl * TB_H * TB_W)), "l"(reinterpret_cast<uint64_t>(&mapM)), "r"(tx * TT - 8),
                "r"(pl * plane_rows + ty * TT - K), "r"(farn_smem_u32(bar)) : "memory");
    };

    int t = blockIdx.x;
    if (tid == 0 && t < ntiles) request(t);
    uint32_t parity = 0;
    for (; t < ntiles; t += gridDim.x) {
        const int ty = t / tiles_x, tx = t - ty * tiles_x;
        const int x0 = tx * TT, y0 = ty * TT;
        farn_mbar_wait(bar, parity);
        parity ^= 1;

        // ---- replicate borders: patch cells whose coordinates clamp (zero-filled or foreign rows from TMA) ----
        if (x0 - K < 0 || y0 - K < 0 || x0 + TT + K > cols || y0 + TT + K > rows) {
            for (int e = tid; e < 5 * TB_H * TSW; e += TNT) {
                const int pl = e / (TB_H * TSW);
                const int rem = e - pl * (TB_H * TSW);
                const int r = rem / TSW, i = rem - r * TSW;
                const int y = y0 - K + r, x = x0 - K + i;
                const int cy = clampi(y, 0, rows - 1), cx = clampi(x, 0, cols - 1);
                if (cy != y || cx != x) {
                    float *P = inbuf + pl * TB_H * TB_W;
                    P[r * TB_W + i + 2] = P[(cy - (y0 - K)) * TB_W + (cx - (x0 - K)) + 2];
                }
            }
            __syncthreads();
        }

        // ---- vertical pass from shared memory: task = (16-row strip, plane, column) ----
        for (int task = tid; task < 4 * 5 * TSW; task += TNT) {
            const int strip = task / (5 * TSW);
            const int rem = task - strip * (5 * TSW);
            const int pl = rem / TSW, i = rem - pl * TSW;
            const float *col = inbuf + (pl * TB_H + strip * 16) * TB_W + i + 2;
            float v[16 + 2 * K];
#pragma unroll
            for (int q = 0; q < 16 + 2 * K; ++q) v[q] = col[q * TB_W];
            float *dst = sums + (pl * TT + strip * 16) * TSW + i;
            if (GAUSS) {
#pragma unroll
                for (int o = 0; o < 16; ++o) {
                    float acc = v[o + K] * gk[0];
#pragma unroll
                    for (int j = 1; j <= K; ++j) acc = acc + (v[o + K - j] + v[o + K + j]) * gk[j];
                    dst[o * TSW] = acc;
                }
            } else {
                float acc = box_first<2 * K + 1>(v);
                dst[0] = acc;
#pragma unroll
                for (int o = 1; o < 16; ++o) {
                    acc = acc + (v[o + 2 * K] - v[o - 1]);
                    dst[o * TSW] = acc;
                }
            }
        }
        __syncthreads();  // sums complete, inbuf free

        const int tn = t + gridDim.x;
        if (tid == 0 && tn < ntiles) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            request(tn);
        }

        // ---- horizontal pass + 2x2 solve + matrix update, 4 pixels per task (as k_farn_iter_fast) ----
#pragma unroll 1
        for (int task = tid; task < TT * (TT / 4); task += TNT) {
            const int r = task / (TT / 4), q = task - r * (TT / 4);
            const int y = y0 + r, x = x0 + 4 * q;
            if (y >= rows || x >= cols) continue;
            float res[5][4];
#pragma unroll
            for (int pl = 0; pl < 5; ++pl) {
                const float *row = sums + (pl * TT + r) * TSW + 4 * q;
                float w[4 + 2 * K + 2];
#pragma unroll
                for (int c = 0; c < (4 + 2 * K + 3) / 4; ++c) {
                    const float4 tq = *reinterpret_cast<const float4 *>(row + 4 * c);
                    w[4 * c] = tq.x;
                    w[4 * c + 1] = tq.y;
                    if (4 * c + 2 < 4 + 2 * K + 2) w[4 * c + 2] = tq.z;
                    if (4 * c + 3 < 4 + 2 * K + 2) w[4 * c + 3] = tq.w;
                }
                if (GAUSS) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float acc = w[e + K] * gk[0];
#pragma unroll
                        for (int i = 1; i <= K; ++i) acc = acc + (w[e + K - i] + w[e + K + i]) * gk[i];
                        res[pl][e] = acc;
                    }
                } else {
                    float acc = box_first<2 * K + 1>(w);
                    res[pl][0] = acc * box_inv;
#pragma unroll
                    for (int e = 1; e < 4; ++e) {
                        acc = acc + (w[e + 2 * K] - w[e - 1]);
                        res[pl][e] = acc * box_inv;
                    }
                }
            }
            float fx[4], fy[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float g11 = res[0][e], g12 = res[1][e], g22 = res[2][e], h1 = res[3][e], h2 = res[4][e];
                const float detInv = 1.f / (g11 * g22 - g12 * g12 + 1e-3f);
                fx[e] = (g11 * h2 - g12 * h1) * detInv;
                fy[e] = (g22 * h1 - g12 * h2) * detInv;
            }
            const bool full = x + 3 < cols;
            if (write_flow) {
                if (full) {
                    *reinterpret_cast<float4 *>(&flowx.at(y, x)) = make_float4(fx[0], fx[1], fx[2], fx[3]);
                    *reinterpret_cast<float4 *>(&flowy.at(y, x)) = make_float4(fy[0], fy[1], fy[2], fy[3]);
                } else {
                    for (int e = 0; e < 4 && x + e < cols; ++e) {
                        flowx.at(y, x + e) = fx[e];
                        flowy.at(y, x + e) = fy[e];
                    }
                }
            }
            if (update_matrices) {
                float m[4][5];
                farn_update_matrices_quad(R0, R1, rows, cols, x, y, fx, fy, m);
#pragma unroll
                for (int pl = 0; pl < 5; ++pl) {
                    if (full) {
                        *reinterpret_cast<float4 *>(&Mout.at(pl, y, x)) = make_float4(m[0][pl], m[1][pl], m[2][pl], m[3][pl]);
                    } else {
                        for (int e = 0; e < 4 && x + e < cols; ++e) Mout.at(pl, y, x + e) = m[e][pl];
                    }
                }
            }
        }
        __syncthreads();  // every warp is done with `sums` before the next tile's vertical pass overwrites it
    }
}

// ------------------------------------------------------------------------------------------
struct FLevel {
    int rows = 0, cols = 0;
    double scale = 1.0;
    int ksize = 3;         // pyramid pre-blur size (smoothSize)
    size_t taps_off = 0;   // offset (floats) of the half kernel in the device table
    Plane img[2];          // level image, both frames (fastPyramids: pyramid level)
    Plane fx, fy;          // flow at this level
};

class FarnebackEngine : public b2f_handle {
public:
    explicit FarnebackEngine(const b2f_farneback_params &p) : P(p) { algo = ALGO_FARNEBACK; }
    b2f_farneback_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    const char *default_name() const override { return "DenseOpticalFlow.FarnebackOpticalFlow"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"farn_iter", "farn_polyexp", "farn_level_image", "farn_update_matrices0",
                                  "farn_flow_init"};
        return (cls >= 0 && cls < 5) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        Layout L;
        std::vector<float> tabs;
        return layout(rows, cols, true, L, tabs);
    }
    bool reads_flow() const override { return (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) != 0; }

private:
    struct Layout {
        int rows = 0, cols = 0;
        b2f_farneback_params P{};
        std::vector<FLevel> levels;  // index k = pyramid level (0 = full res)
        Plane frames[2];
        Plane vbuf[2];
        Stack5 R[2], M[2];
        float *tabs_dev = nullptr;
        size_t tabs_count = 0;
        size_t win_taps_off = 0;  // GAUSSIAN flag: window kernel
        PolyTabs poly;
    };
    Layout L_;

    // the whole fixed schedule between the conversion of the caller's frames and the final merge, as one CUDA graph
    struct GraphKey {
        int rows, cols;
        b2f_farneback_params P;
        EngineKnobs knobs;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && same_knobs(knobs, o.knobs) && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;
    void solve(Ctx &c);

    size_t layout(int rows, int cols, bool counting, Layout &L, std::vector<float> &tabs);
    cudaError_t ensure_workspace(int rows, int cols, cudaStream_t s);
    std::vector<float> tabs_host_;  // source of the asynchronous table upload
};

size_t FarnebackEngine::layout(int rows, int cols, bool counting, Layout &L, std::vector<float> &tabs) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.rows = rows;
    L.cols = cols;
    L.P = P;
    L.levels.clear();
    tabs.clear();

    // crop levels, farneback.cpp:333-340
    double scale = 1;
    int cropped = 0;
    for (; cropped < P.num_levels; cropped++) {
        scale *= P.pyr_scale;
        if (cols * scale < MIN_SIZE || rows * scale < MIN_SIZE) break;
    }
    L.frames[0] = A.plane(rows, cols);
    L.frames[1] = A.plane(rows, cols);
    int max_lrows = 0;
    int pr = rows, pc = cols;
    for (int k = 0; k <= cropped; ++k) {
        FLevel lv;
        scale = 1;
        for (int i = 0; i < k; i++) scale *= P.pyr_scale;
        lv.scale = scale;
        const double sigma = (1. / scale - 1) * 0.5;  // farneback.cpp:372-374
        int smooth = cv_round(sigma * 5) | 1;
        smooth = smooth > 3 ? smooth : 3;
        lv.ksize = smooth;
        if (P.fast_pyramids) {  // pyrDown sizes, pyramids.cpp:66-93
            if (k > 0) {
                pr = (pr + 1) / 2;
                pc = (pc + 1) / 2;
            }
            lv.rows = pr;
            lv.cols = pc;
        } else {
            lv.cols = cv_round(cols * scale);
            lv.rows = cv_round(rows * scale);
            if (lv.cols < 1) lv.cols = 1;
            if (lv.rows < 1) lv.rows = 1;
            std::vector<float> gk;
            gaussian_kernel(smooth, sigma, gk);
            lv.taps_off = tabs.size();
            for (int i = smooth / 2; i < smooth; ++i) tabs.push_back(gk[i]);
        }
        if (k == 0 && P.fast_pyramids) {
            lv.img[0] = L.frames[0];
            lv.img[1] = L.frames[1];
        } else {
            lv.img[0] = A.plane(lv.rows, lv.cols);
            lv.img[1] = A.plane(lv.rows, lv.cols);
        }
        lv.fx = A.plane(lv.rows, lv.cols);
        lv.fy = A.plane(lv.rows, lv.cols);
        if (lv.rows > max_lrows) max_lrows = lv.rows;
        L.levels.push_back(lv);
    }
    if (P.flags & B2F_OPTFLOW_FARNEBACK_GAUSSIAN) {  // farneback.cpp:460-464
        std::vector<float> gk;
        gaussian_kernel(P.win_size, static_cast<double>(static_cast<float>(P.win_size / 2 * 0.3f)), gk);
        L.win_taps_off = tabs.size();
        for (int i = P.win_size / 2; i < P.win_size; ++i) tabs.push_back(gk[i]);
    }
    if (tabs.empty()) tabs.push_back(0.f);
    L.tabs_count = tabs.size();
    if (!P.fast_pyramids) {
        L.vbuf[0] = A.plane(2 * max_lrows, cols);
        L.vbuf[1] = A.plane(2 * max_lrows, cols);
    }
    for (int i = 0; i < 2; ++i) {
        // R gets one spare row: the quad / spread gathers point a pixel without a bilinear cell at (0, 0) and still
        // load its row below, which on a one-row level lies one row past plane 4 (the loaded values are discarded)
        Plane r = A.plane(5 * rows + 1, cols), m = A.plane(5 * rows, cols);
        L.R[i] = Stack5{r.p, r.pitch, rows};
        L.M[i] = Stack5{m.p, m.pitch, rows};
    }
    L.tabs_dev = static_cast<float *>(A.bytes(sizeof(float) * tabs.size()));
    return A.used();
}

cudaError_t FarnebackEngine::ensure_workspace(int rows, int cols, cudaStream_t s) {
    if (L_.rows == rows && L_.cols == cols && same_params(L_.P, P) && arena.capacity() > 0)
        return cudaSuccess;
    Layout tmp;
    std::vector<float> tabs;
    const size_t need = layout(rows, cols, true, tmp, tabs);
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    // Re-layout of a live arena (new size or parameters on the same handle): kernels of the previous call may still be
    // reading it on the caller's stream, and the table upload below must be ordered against them too.
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return e;
    layout(rows, cols, false, L_, tabs);
    if (!prepare_poly_tabs(P.poly_n, P.poly_sigma, L_.poly)) return cudaErrorInvalidValue;
    // one-time table upload on the call's stream (the reference re-uploads __constant__ tables every call); the host copy
    // lives in the handle so the asynchronous copy never reads a dead buffer
    tabs_host_ = tabs;
    return cudaMemcpyAsync(L_.tabs_dev, tabs_host_.data(), sizeof(float) * tabs_host_.size(), cudaMemcpyHostToDevice, s);
}

int FarnebackEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    // preconditions: farneback.cpp:173-174,181-182,316-317
    if (!(I0->type == B2F_8UC1 || I0->type == B2F_32FC1)) return B2F_UNSUPPORTED_TYPE;
    if (I0->type != I1->type) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    if (!(P.poly_n == 5 || P.poly_n == 7)) return B2F_BAD_ARG;
    if (P.fast_pyramids && !(std::abs(P.pyr_scale - 0.5) < 1e-6)) return B2F_BAD_ARG;
    if (P.num_levels < 0 || P.num_iters < 0 || P.win_size < 1 || (P.win_size & 1) == 0) return B2F_BAD_ARG;
    if (!(P.pyr_scale > 0.0 && P.pyr_scale < 1.0)) return B2F_BAD_ARG;
    const size_t es = I0->type == B2F_8UC1 ? 1 : 4;
    if (I0->step < I0->cols * es || I1->step < I1->cols * es || !flow_step_ok(flow)) return B2F_BAD_ARG;

    const int rows = I0->rows, cols = I0->cols;
    Ctx c = make_ctx(s);
    c.check(ensure_workspace(rows, cols, s));
    if (!c.ok()) return finish(c, s);
    static DeviceOnce attrs;
    attrs.run(c, [&] {
        const int bytes = (int)(sizeof(float) * 5 * FT_H * (FT_W + 12));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, false, true, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, false, true, 256, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, false, true, 256, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        c.check(cudaFuncSetAttribute(k_farn_iter_fast<6, false, true, 256, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes + 8 * 1024));
        c.check(cudaFuncSetAttribute(k_farn_iter_tma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FARN_TMA_SMEM));
        c.check(cudaFuncSetAttribute(k_farn_iter_tma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FARN_TMA_SMEM));
    });
    Layout &L = L_;
    const int top = static_cast<int>(L.levels.size()) - 1;
    stats.levels = top + 1;
    stats.iterations_run = 0;
    active_paths.assign(top + 1, 0.0);

    const ImageView v0{I0->data, I0->step, rows, cols, I0->type};
    const ImageView v1{I1->data, I1->step, rows, cols, I1->type};
    const ImageView vf = flow_view(flow, rows, cols);
    const dim3 block(32, 8);

    convert_pair(c, CLS_IMG, v0, v1, L.frames[0], L.frames[1], 1.0f);  // convertTo(CV_32F), farneback.cpp:342-345
    if (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) split_flow(c, CLS_FLOW, vf, L.levels[0].fx, L.levels[0].fy);

    // Every launch below works on arena planes only, so the schedule is captured once per (size, parameters) and
    // replayed: one graph launch instead of ~90 kernel launches per pair (the coarse levels are launch-bound).
    const bool want_graph = knobs.use_graph && !profiling && s != nullptr;
    if (want_graph) {
        graph_.run(*this, c, s, GraphKey{rows, cols, P, knobs, L.frames[0].p}, [&](Ctx &g) { solve(g); });
    } else {
        solve(c);
    }

    merge_flow(c, CLS_FLOW, L.levels[0].fx, L.levels[0].fy, vf);  // farneback.cpp:197-198
    return finish(c, s);
}

void FarnebackEngine::solve(Ctx &c) {
    Layout &L = L_;
    const int rows = L.rows, cols = L.cols;
    const int top = static_cast<int>(L.levels.size()) - 1;
    const dim3 block(32, 8);
    if (P.fast_pyramids) {
        for (int k = 1; k <= top; ++k)
            for (int i = 0; i < 2; ++i)
                pyr_down(c, CLS_IMG, L.levels[k - 1].img[i], L.levels[k - 1].rows, L.levels[k - 1].cols,
                         L.levels[k].img[i], L.levels[k].rows, L.levels[k].cols);
    }

    const int khalf = P.win_size / 2;
    const float box_inv = 1.f / ((1 + 2 * khalf) * (1 + 2 * khalf));
    const bool gauss = (P.flags & B2F_OPTFLOW_FARNEBACK_GAUSSIAN) != 0;
    const float *win_taps = L.tabs_dev + L.win_taps_off;

    for (int k = top; k >= 0; --k) {
        FLevel &lv = L.levels[k];
        const int h = lv.rows, w = lv.cols;
        const double npx = (double)h * w;
        const dim3 grid(div_up(w, 32), div_up(h, 8));

        // ---- flow initialisation, farneback.cpp:396-417 ----
        if (k == top) {
            if (P.flags & B2F_OPTFLOW_USE_INITIAL_FLOW) {
                if (k > 0)
                    resize_linear_pair(c, CLS_FLOW, L.levels[0].fx, L.levels[0].fy, rows, cols, lv.fx, lv.fy, h, w,
                                       inv_scale_from_sizes(cols, w), inv_scale_from_sizes(rows, h),
                                       static_cast<float>(lv.scale));
            } else {
                fill_plane(c, lv.fx, h, w, 0.f);
                fill_plane(c, lv.fy, h, w, 0.f);
            }
        } else {
            const FLevel &pv = L.levels[k + 1];
            resize_linear_pair(c, CLS_FLOW, pv.fx, pv.fy, pv.rows, pv.cols, lv.fx, lv.fy, h, w,
                               inv_scale_from_sizes(pv.cols, w), inv_scale_from_sizes(pv.rows, h),
                               static_cast<float>(1. / P.pyr_scale));
        }

        // ---- level images ----
        if (!P.fast_pyramids) {
            const int kh = lv.ksize / 2;
            const float *taps = L.tabs_dev + lv.taps_off;
            const int identity = (h == rows && w == cols) ? 1 : 0;  // resize.cpp:90-94 copy path
            const float inv_fx = inv_scale_from_sizes(cols, w), inv_fy = inv_scale_from_sizes(rows, h);
            const dim3 gv(div_up(cols, 256), 2 * h, 2);
            if (knobs.aux_path == 6) {  // the round-1 kernel: one column per thread
                B2F_LAUNCH(c, CLS_IMG, 2.0 * 4.0 * ((double)rows * cols + 2.0 * h * cols), k_farn_blur_v, gv, dim3(256), 0,
                           L.frames[0], L.frames[1], rows, cols, L.vbuf[0], L.vbuf[1], h, inv_fy, taps, kh, identity);
            } else {
                // odd rows of the staging buffer are only read with a non-zero weight when y / fy has a fractional part
                const int ystep = (identity || inv_fy == std::floor(inv_fy)) ? 2 : 1;
                const dim3 gv4(div_up(cols, 1024), ystep == 2 ? h : 2 * h, 2);
                B2F_LAUNCH(c, CLS_IMG, 2.0 * 4.0 * ((double)rows * cols + 2.0 * h * cols), k_farn_blur_v4, gv4, dim3(256), 0,
                           L.frames[0], L.frames[1], rows, cols, L.vbuf[0], L.vbuf[1], h, inv_fy, taps, kh, identity, ystep);
            }
            const dim3 gh(div_up(w, 32), div_up(h, 8), 2);
            B2F_LAUNCH(c, CLS_IMG, 2.0 * 4.0 * (2.0 * h * cols + npx), k_farn_blur_h_resize, gh, block, 0, L.vbuf[0],
                       L.vbuf[1], rows, cols, lv.img[0], lv.img[1], h, w, inv_fx, inv_fy, taps, kh, identity);
        }

        // ---- polynomial expansion of both frames ----
        Stack5 R0{L.R[0].p, plane_pitch(w), h}, R1{L.R[1].p, plane_pitch(w), h};
        Stack5 Ma{L.M[0].p, plane_pitch(w), h}, Mb{L.M[1].p, plane_pitch(w), h};
        {
            const dim3 gp(div_up(w, 32), div_up(h, 8), 2), gpf(div_up(w, 64), div_up(h, 32), 2);
            const double bytes = 2.0 * 24.0 * npx;
            Plane a{lv.img[0].p, lv.img[0].pitch}, b{lv.img[1].p, lv.img[1].pitch};
            if (knobs.aux_path == 6) {  // the round-1 kernel (one vertical-pass evaluation per output)
                if (P.poly_n == 5)
                    B2F_LAUNCH(c, CLS_POLY, bytes, k_farn_polyexp<5>, gp, block, 0, a, b, R0, R1, h, w, L.poly);
                else
                    B2F_LAUNCH(c, CLS_POLY, bytes, k_farn_polyexp<7>, gp, block, 0, a, b, R0, R1, h, w, L.poly);
            } else if (P.poly_n == 5) {
                B2F_LAUNCH(c, CLS_POLY, bytes, k_farn_polyexp_fast<5>, gpf, block, 0, a, b, R0, R1, h, w, L.poly);
            } else {
                B2F_LAUNCH(c, CLS_POLY, bytes, k_farn_polyexp_fast<7>, gpf, block, 0, a, b, R0, R1, h, w, L.poly);
            }
        }

        // ---- initial matrices, then the fused iterations ----
        B2F_LAUNCH(c, CLS_UPD0, 68.0 * npx, k_farn_update_matrices, grid, block, 0, lv.fx, lv.fy, R0, R1, Ma, h, w);
        const dim3 gi(div_up(w, IT_TW), div_up(h, IT_TH));
        const size_t smem = sizeof(float) * 5 * IT_TH * (IT_TW + 2 * khalf);
        const bool fast6 = khalf == 6 && knobs.kernel_path != 1;
        const dim3 gf(div_up(w, FT_W), div_up(h, FT_H));
        const size_t smem_fast = sizeof(float) * 5 * FT_H * (FT_W + 12);
        // Coarse levels leave most SMs idle and are bound by each thread's chain of dependent round trips (three
        // column tasks, two quad tasks): 512 threads per tile halve that chain.  Same arithmetic, same bits.
        const bool wide_blocks = (int)(gf.x * gf.y) <= sm_count() && knobs.fused_iters != 256;
        // opt-in persistent TMA kernel (kernel_path 3) on levels with at least two waves of 64x64 tiles
        const int tma_tx = div_up(w, TT), tma_ty = div_up(h, TT);
        bool use_tma = knobs.kernel_path == 3 && khalf == 6 && tma_tx * tma_ty >= 2 * sm_count();
        alignas(64) CUtensorMap mapA, mapB;
        if (use_tma) {
            const uint64_t pitch_b = sizeof(float) * (uint64_t)plane_pitch(w);
            use_tma = tma_encode_2d_f32(&mapA, Ma.p, (uint64_t)w, 5ull * h, pitch_b, TB_W, TB_H) &&
                      tma_encode_2d_f32(&mapB, Mb.p, (uint64_t)w, 5ull * h, pitch_b, TB_W, TB_H);
        }
        {  // the kernel the loop below launches (same branch order), reported as active path k
            const bool quad = knobs.kernel_path != 2;
            int path = B2F_FARN_PATH_GENERIC;
            if (use_tma) path = B2F_FARN_PATH_TMA;
            else if (fast6 && !quad) path = B2F_FARN_PATH_FAST;
            else if (fast6 && gauss) path = B2F_FARN_PATH_QUAD;
            else if (fast6 && wide_blocks) path = B2F_FARN_PATH_QUAD_WIDE;
            else if (fast6 && knobs.aux_path == 3) path = B2F_FARN_PATH_QUAD_R80;
            else if (fast6 && knobs.aux_path == 5) path = B2F_FARN_PATH_QUAD_TRANSPOSED;
            else if (fast6 && knobs.aux_path == 4) path = B2F_FARN_PATH_QUAD_R64;
            else if (fast6) path = B2F_FARN_PATH_QUAD;
            active_paths[k] = P.num_iters > 0 ? path : 0;
        }
        bool a_is_input = true;
        for (int i = 0; i < P.num_iters; ++i) {
            const int upd = i < P.num_iters - 1;  // farneback.cpp:468-470
            const int wflow = !upd;
            const double bytes = npx * (20.0 + (upd ? 60.0 : 0.0) + (wflow ? 8.0 : 0.0));
            if (use_tma) {
                const int ntiles = tma_tx * tma_ty;
                const dim3 gt(ntiles < sm_count() ? ntiles : sm_count());
                const CUtensorMap &mapIn = a_is_input ? mapA : mapB;
                if (gauss)
                    B2F_LAUNCH(c, CLS_ITER, bytes, k_farn_iter_tma<true>, gt, dim3(TNT), FARN_TMA_SMEM, mapIn, Mb, R0, R1,
                               lv.fx, lv.fy, h, w, h, box_inv, win_taps, upd, wflow, tma_tx, ntiles);
                else
                    B2F_LAUNCH(c, CLS_ITER, bytes, k_farn_iter_tma<false>, gt, dim3(TNT), FARN_TMA_SMEM, mapIn, Mb, R0, R1,
                               lv.fx, lv.fy, h, w, h, box_inv, win_taps, upd, wflow, tma_tx, ntiles);
            } else if (fast6) {
                const bool quad = knobs.kernel_path != 2;
                if (gauss && quad)
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, true, true>), gf, dim3(256), smem_fast, Ma, Mb, R0,
                               R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else if (gauss)
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, true, false>), gf, dim3(256), smem_fast, Ma, Mb, R0,
                               R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else if (quad && wide_blocks)
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, false, true, 512>), gf, dim3(512), smem_fast, Ma, Mb,
                               R0, R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else if (quad && knobs.aux_path == 3)  // 80 registers: 3 blocks / SM
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, false, true, 256, 3>), gf, dim3(256), smem_fast, Ma, Mb,
                               R0, R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else if (quad && knobs.aux_path == 5)  // lane-transposed R1 gather
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, false, true, 256, 2, true>), gf, dim3(256),
                               smem_fast + 8 * 1024, Ma, Mb, R0, R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else if (quad && knobs.aux_path == 4)  // 64 registers: 4 blocks / SM
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, false, true, 256, 4>), gf, dim3(256), smem_fast, Ma, Mb,
                               R0, R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else if (quad)
                    // 128 registers, 2 blocks / SM.  The kernel waits on its gathers; capping it at 80 or 64 registers
                    // buys occupancy with spills and lost instruction-level parallelism (aux_path 3 / 4 keep those
                    // variants, bit-identical)
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, false, true>), gf, dim3(256), smem_fast, Ma, Mb, R0,
                               R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
                else
                    B2F_LAUNCH(c, CLS_ITER, bytes, (k_farn_iter_fast<6, false, false>), gf, dim3(256), smem_fast, Ma, Mb,
                               R0, R1, lv.fx, lv.fy, h, w, box_inv, win_taps, upd, wflow);
            } else if (gauss)
                B2F_LAUNCH(c, CLS_ITER, bytes, k_farn_iter<true>, gi, dim3(256), smem, Ma, Mb, R0, R1, lv.fx, lv.fy, h,
                           w, khalf, box_inv, win_taps, upd, wflow);
            else
                B2F_LAUNCH(c, CLS_ITER, bytes, k_farn_iter<false>, gi, dim3(256), smem, Ma, Mb, R0, R1, lv.fx, lv.fy,
                           h, w, khalf, box_inv, win_taps, upd, wflow);
            Stack5 t = Ma;
            Ma = Mb;
            Mb = t;
            a_is_input = !a_is_input;
            c.stats->iterations_run++;
        }
    }
}

int FarnebackEngine::set_param(int id, double v) {
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

int FarnebackEngine::get_param(int id, double *v) const {
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

void b2f_farneback_default_params(b2f_farneback_params *p) {
    if (!p) return;
    p->num_levels = 5;
    p->pyr_scale = 0.5;
    p->fast_pyramids = 0;
    p->win_size = 13;
    p->num_iters = 10;
    p->poly_n = 5;
    p->poly_sigma = 1.1;
    p->flags = 0;
}

int b2f_farneback_create(const b2f_farneback_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_farneback_params d;
    b2f_farneback_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::FarnebackEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
