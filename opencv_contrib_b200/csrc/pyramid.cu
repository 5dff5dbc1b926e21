// pyramid.cu -- the small data-movement kernels on either side of the solvers: type conversion,
// bilinear pyramid resize (+ fused flow rescale), pyrDown, planar<->interleaved flow.
// Each is a single coalesced pass; 32x8 thread blocks over the destination.
#include "common.cuh"

namespace b2f {

namespace {

struct Pair {
    Plane a, b;
};

template <typename T>
__global__ void k_convert_pair(const T *__restrict__ sa, const T *__restrict__ sb, size_t step_a, size_t step_b,
                               Plane da, Plane db, int rows, int cols, float scale) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const bool second = blockIdx.z != 0;
    const char *base = reinterpret_cast<const char *>(second ? sb : sa) + (size_t)y * (second ? step_b : step_a);
    const float v = static_cast<float>(reinterpret_cast<const T *>(base)[x]);
    (second ? db : da).at(y, x) = v * scale;
}

// cv::cuda::resize INTER_LINEAR float C1: src = dst * scale, x2/y2 reads clamped, weights from the
// unclamped neighbours (cudawarping/src/cuda/resize.cu:234-269).  `mul` fuses the flow rescale.  The reference's
// `out = out + src * (w_x * w_y)` is written out as the rounding nvcc contracts it into: each weight product rounded on
// its own, then one fused multiply-add per tap, the first one onto +0.  The remaining plain expressions here and in
// k_convert_pair / k_copy_plane are single rounded operations with nothing to contract.
__device__ __forceinline__ float resize_sample(const Plane &s, int srows, int scols, int dx, int dy, float inv_fx,
                                               float inv_fy) {
    const float src_x = dx * inv_fx;
    const float src_y = dy * inv_fy;
    const int x1 = __float2int_rd(src_x);
    const int y1 = __float2int_rd(src_y);
    const int x2 = x1 + 1, y2 = y1 + 1;
    const int x1r = min(x1, scols - 1), y1r = min(y1, srows - 1);  // defensive; x1 <= scols-1 by construction
    const int x2r = min(x2, scols - 1), y2r = min(y2, srows - 1);
    const float wx2 = x2 - src_x, wx1 = src_x - x1;
    const float wy2 = y2 - src_y, wy1 = src_y - y1;
    float out = 0.f;
    out = __fmaf_rn(__ldg(&s.at(y1r, x1r)), __fmul_rn(wx2, wy2), out);
    out = __fmaf_rn(__ldg(&s.at(y1r, x2r)), __fmul_rn(wx1, wy2), out);
    out = __fmaf_rn(__ldg(&s.at(y2r, x1r)), __fmul_rn(wx2, wy1), out);
    out = __fmaf_rn(__ldg(&s.at(y2r, x2r)), __fmul_rn(wx1, wy1), out);
    return out;
}

__global__ void k_resize_linear(Plane sa, Plane sb, int srows, int scols, Plane da, Plane db, int drows, int dcols,
                                float inv_fx, float inv_fy, float mul, int apply_mul) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dcols || y >= drows) return;
    const bool second = blockIdx.z != 0;
    float v = resize_sample(second ? sb : sa, srows, scols, x, y, inv_fx, inv_fy);
    if (apply_mul) v = v * mul;
    (second ? db : da).at(y, x) = v;
}

__global__ void k_copy_plane(Plane sa, Plane sb, Plane da, Plane db, int rows, int cols, float mul, int apply_mul) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const bool second = blockIdx.z != 0;
    float v = (second ? sb : sa).at(y, x);
    if (apply_mul) v = v * mul;
    (second ? db : da).at(y, x) = v;
}

__global__ void k_merge(Plane u, Plane v, float *__restrict__ flow, size_t step, int rows, int cols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    float2 *row = reinterpret_cast<float2 *>(reinterpret_cast<char *>(flow) + (size_t)y * step);
    row[x] = make_float2(u.at(y, x), v.at(y, x));
}

__global__ void k_split(const float *__restrict__ flow, size_t step, Plane u, Plane v, int rows, int cols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const float2 *row = reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(flow) + (size_t)y * step);
    const float2 f = row[x];
    u.at(y, x) = f.x;
    v.at(y, x) = f.y;
}

// BORDER_REFLECT101 index (cv::cuda::device::BrdReflect101): -1 -> 1, n -> n-2.
__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        if (i >= n) i = 2 * n - 2 - i;
    }
    return i;
}

// One [1 4 6 4 1]/16 tap chain with its roundings spelled out: the first two products summed with one rounding, then
// one fused multiply-add per remaining tap.  This is the instruction sequence nvcc contracts the plain expression
// into; written out, it no longer depends on the compiler, and the models (oracle/denselk_model.py, .c) restate it.
// Products by 0.0625 and 0.25 are exact, so only the 0.375 tap and the sums round.
__device__ __forceinline__ float pyr_tap5(float a, float b, float c, float d, float e) {
    float s = __fmaf_rn(a, 0.0625f, __fmul_rn(b, 0.25f));
    s = __fmaf_rn(c, 0.375f, s);
    s = __fmaf_rn(d, 0.25f, s);
    return __fmaf_rn(e, 0.0625f, s);
}

// cv::cuda::pyrDown (cudawarping/src/cuda/pyr_down.cu:55-173): horizontal 5-tap [1 4 6 4 1] on the
// five source rows 2y-2..2y+2 (reflect101), then vertical 5-tap, /256.  Same operation order:
// row sums first (sum over the 5 rows weighted), then across columns, scaled by 1/256 at the end.
template <bool ROUND_U8>
__global__ void k_pyr_down(Plane s, int srows, int scols, Plane d, int drows, int dcols) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dcols || y >= drows) return;
    const int sy = 2 * y, sx = 2 * x;
    int ry[5], rx[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        ry[k] = reflect101(sy - 2 + k, srows);
        rx[k] = reflect101(sx - 2 + k, scols);
    }
    // vertical 5-tap per source column, then horizontal 5-tap, each in the reference's left-to-right
    // order 0.0625*a + 0.25*b + 0.375*c + 0.25*d + 0.0625*e (pyr_down.cu:68-73,139-144), rounded as pyr_tap5 says
    float col[5];
#pragma unroll
    for (int i = 0; i < 5; ++i)
        col[i] = pyr_tap5(__ldg(&s.at(ry[0], rx[i])), __ldg(&s.at(ry[1], rx[i])), __ldg(&s.at(ry[2], rx[i])),
                          __ldg(&s.at(ry[3], rx[i])), __ldg(&s.at(ry[4], rx[i])));
    float out = pyr_tap5(col[0], col[1], col[2], col[3], col[4]);
    // 8-bit pyramids: saturate_cast<uchar>(sum) rounds half to even (pyr_down.cu:172)
    if (ROUND_U8) out = rintf(fminf(fmaxf(out, 0.f), 255.f));
    d.at(y, x) = out;
}

}  // namespace

static dim3 grid2d(int cols, int rows, int z) { return dim3(div_up(cols, 32), div_up(rows, 8), z); }

void convert_pair(Ctx &c, int cls, const ImageView &a, const ImageView &b, Plane da, Plane db, float scale) {
    const dim3 block(32, 8);
    const dim3 grid = grid2d(a.cols, a.rows, 2);
    const double bytes = 2.0 * a.rows * a.cols * ((a.type == B2F_8UC1 ? 1 : 4) + 4);
    if (a.type == B2F_8UC1) {
        B2F_LAUNCH(c, cls, bytes, k_convert_pair<unsigned char>, grid, block, 0,
                   static_cast<const unsigned char *>(a.data), static_cast<const unsigned char *>(b.data), a.step,
                   b.step, da, db, a.rows, a.cols, scale);
    } else {
        B2F_LAUNCH(c, cls, bytes, k_convert_pair<float>, grid, block, 0, static_cast<const float *>(a.data),
                   static_cast<const float *>(b.data), a.step, b.step, da, db, a.rows, a.cols, scale);
    }
}

void resize_linear_pair(Ctx &c, int cls, Plane sa, Plane sb, int srows, int scols, Plane da, Plane db, int drows,
                        int dcols, float inv_fx, float inv_fy, float mul) {
    const dim3 block(32, 8);
    const dim3 grid = grid2d(dcols, drows, 2);
    const double bytes = 2.0 * 4.0 * ((double)drows * dcols + (double)srows * scols);
    const int apply_mul = mul != 1.0f;
    if (drows == srows && dcols == scols) {  // resize.cpp:90-94: equal size -> copyTo
        B2F_LAUNCH(c, cls, bytes, k_copy_plane, grid, block, 0, sa, sb, da, db, drows, dcols, mul, apply_mul);
    } else {
        B2F_LAUNCH(c, cls, bytes, k_resize_linear, grid, block, 0, sa, sb, srows, scols, da, db, drows, dcols, inv_fx,
                   inv_fy, mul, apply_mul);
    }
}

void resize_linear_one(Ctx &c, int cls, Plane s, int srows, int scols, Plane d, int drows, int dcols, float inv_fx,
                       float inv_fy, float mul) {
    const dim3 block(32, 8);
    const dim3 grid = grid2d(dcols, drows, 1);
    const double bytes = 4.0 * ((double)drows * dcols + (double)srows * scols);
    const int apply_mul = mul != 1.0f;
    if (drows == srows && dcols == scols) {
        B2F_LAUNCH(c, cls, bytes, k_copy_plane, grid, block, 0, s, s, d, d, drows, dcols, mul, apply_mul);
    } else {
        B2F_LAUNCH(c, cls, bytes, k_resize_linear, grid, block, 0, s, s, srows, scols, d, d, drows, dcols, inv_fx,
                   inv_fy, mul, apply_mul);
    }
}

void merge_flow(Ctx &c, int cls, Plane u, Plane v, const ImageView &flow) {
    if (flow.data2) {  // planar output: two pitched device-to-device copies
        if (!c.ok()) return;
        const size_t w = sizeof(float) * (size_t)flow.cols;
        c.check(cudaMemcpy2DAsync(flow.data, flow.step, u.p, sizeof(float) * (size_t)u.pitch, w, flow.rows,
                                  cudaMemcpyDeviceToDevice, c.stream));
        c.check(cudaMemcpy2DAsync(flow.data2, flow.step2, v.p, sizeof(float) * (size_t)v.pitch, w, flow.rows,
                                  cudaMemcpyDeviceToDevice, c.stream));
        return;
    }
    const dim3 block(32, 8);
    const dim3 grid = grid2d(flow.cols, flow.rows, 1);
    B2F_LAUNCH(c, cls, 16.0 * flow.rows * flow.cols, k_merge, grid, block, 0, u, v, static_cast<float *>(flow.data),
               flow.step, flow.rows, flow.cols);
}

void split_flow(Ctx &c, int cls, const ImageView &flow, Plane u, Plane v) {
    if (flow.data2) {
        if (!c.ok()) return;
        const size_t w = sizeof(float) * (size_t)flow.cols;
        c.check(cudaMemcpy2DAsync(u.p, sizeof(float) * (size_t)u.pitch, flow.data, flow.step, w, flow.rows,
                                  cudaMemcpyDeviceToDevice, c.stream));
        c.check(cudaMemcpy2DAsync(v.p, sizeof(float) * (size_t)v.pitch, flow.data2, flow.step2, w, flow.rows,
                                  cudaMemcpyDeviceToDevice, c.stream));
        return;
    }
    const dim3 block(32, 8);
    const dim3 grid = grid2d(flow.cols, flow.rows, 1);
    B2F_LAUNCH(c, cls, 16.0 * flow.rows * flow.cols, k_split, grid, block, 0, static_cast<const float *>(flow.data),
               flow.step, u, v, flow.rows, flow.cols);
}

void fill_plane(Ctx &c, Plane p, int rows, int cols, float) {
    (void)cols;
    if (!c.ok()) return;
    c.check(cudaMemsetAsync(p.p, 0, sizeof(float) * (size_t)p.pitch * rows, c.stream));
}

void pyr_down(Ctx &c, int cls, Plane s, int srows, int scols, Plane d, int drows, int dcols) {
    const dim3 block(32, 8);
    const dim3 grid = grid2d(dcols, drows, 1);
    B2F_LAUNCH(c, cls, 4.0 * ((double)srows * scols + (double)drows * dcols), k_pyr_down<false>, grid, block, 0, s, srows,
               scols, d, drows, dcols);
}

void pyr_down_u8(Ctx &c, int cls, Plane s, int srows, int scols, Plane d, int drows, int dcols) {
    const dim3 block(32, 8);
    const dim3 grid = grid2d(dcols, drows, 1);
    B2F_LAUNCH(c, cls, 4.0 * ((double)srows * scols + (double)drows * dcols), k_pyr_down<true>, grid, block, 0, s, srows,
               scols, d, drows, dcols);
}

}  // namespace b2f
