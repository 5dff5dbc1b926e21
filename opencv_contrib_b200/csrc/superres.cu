// superres.cu -- superres's BTV-L1 video super-resolution (cv::superres::createSuperResolution_BTVL1_CUDA,
// modules/superres/src/btv_l1_cuda.cpp, src/cuda/btv_l1_gpu.cu) and the colour / depth conversion of its CUDA optical-flow
// wrappers (src/optical_flow.cpp:440-849, src/input_array_utility.cpp).
//
// Built with -fmad=false: every operator rounds once, in the order oracle/superres_model.c states them.
//
// Per processed frame:
//   k_sr_window  (low resolution)  window frames copied out of the ring, relative motions summed (calcRelativeMotions)
//   k_sr_maps    (high resolution) both motion maps: cubic upscale x scale, p + motion, truncated and clamped to a linear
//                                  nearest-neighbour index; and the cubic upscale of the base frame (the initial estimate)
// Per iteration (one CUDA graph for the whole loop):
//   k_sr_forward (low resolution x K)  sign(src_k - D H M_k hr): the blur evaluated only where the decimation samples it
//   k_sr_update  (high resolution)     hr - tau lambda BTV(hr) + tau sum_k M_k^T H^T D^T sign_k, reading hr as it stood at
//                                      the start of the iteration (the reference's streams join before the update)
#include "common.cuh"

#include <cmath>
#include <cstring>
#include <new>

namespace b2f {
namespace {

constexpr int SR_MAX_K = 2 * B2F_SR_MAX_RADIUS + 1;
constexpr int SR_MAX_BLUR = 31;
constexpr int SR_MAX_BTV_TAPS = 96;  // sum over m = 0..7 of (7 + m + 1) = 92 weights at btvKernelSize 16

enum { CLS_ITER_FORWARD = 0, CLS_ITER_UPDATE = 1, CLS_MAPS = 2, CLS_WINDOW = 3, CLS_INGEST = 4, CLS_OUTPUT = 5 };

// cudafilters' BrdRowReflect101 / BrdColReflect101 as the row and column filters use them (at_low below the image,
// at_high above it)
__host__ __device__ __forceinline__ int reflect101(int x, int n) {
    const int last = n - 1;
    if (x < 0) return abs(x) % n;
    if (x > last) return abs(last - abs(last - x)) % n;
    return x;
}

// core's CubicFilter::bicubicCoeff, Keys a = -0.5
__device__ __forceinline__ float cubic_coeff(float x_) {
    const float x = fabsf(x_);
    if (x <= 1.0f) return x * x * (1.5f * x - 2.5f) + 1.0f;
    if (x < 2.0f) return x * (x * (-0.5f * x + 2.5f) - 4.0f) + 2.0f;
    return 0.0f;
}

__device__ __forceinline__ float diff_sign(float a, float b) { return a > b ? 1.0f : a < b ? -1.0f : 0.0f; }

// PointFilter + BrdReplicate: clamp(__float2int_rz(v)) (NaN -> 0, saturating like the PTX conversion)
__device__ __forceinline__ int nearest_index(float v, int n) { return min(max(__float2int_rz(v), 0), n - 1); }

struct SrGeom {
    int lr_rows, lr_cols, cn, scale, hr_rows, hr_cols;
    int lp;   // pitch (floats) of single-channel low-resolution planes
    int lpc;  // pitch (floats) of interleaved low-resolution frames
    int hpc;  // pitch (floats) of interleaved high-resolution images: hr_cols * cn, unpadded (linear map indices)
    int hp;   // pitch (ints) of high-resolution index planes
    int sp;   // pitch (bytes) of sign planes
    size_t lr_plane, lr_frame, hr_image, hr_index, sign_plane;  // element strides between consecutive planes
};

struct SrWindow {
    int K, base;
    int frame_slot[SR_MAX_K];
    int fwd_slot[SR_MAX_K];  // forwardMotions at(i) for i < end
    int bwd_slot[SR_MAX_K];  // backwardMotions at(i) for i > start
};

struct SrIter {
    float blur[SR_MAX_BLUR + 1];
    float btv[SR_MAX_BTV_TAPS];
    int bk, anchor, ks, K, reg;
    float reg_beta, tau;
};

// ------------------------------------------------------------------------------------------------ ingest / wrappers
// 8UC{1,3,4} -> float, unscaled (GpuMat::convertTo(CV_32F))
__global__ void k_sr_ingest(const uint8_t *src, size_t step, int rows, int cols, int cn, float *dst, int dpitch) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols * cn || y >= rows) return;
    dst[(size_t)y * dpitch + x] = (float)src[(size_t)y * step + x];
}

// cvtColor(BGR2GRAY / BGRA2GRAY) with cudev's 15-bit rule, then convertTo(depth, 1 or 1/255)
__global__ void k_sr_gray(const uint8_t *src, size_t step, int rows, int cols, int cn, void *dst, size_t dstep, int to_f32) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const uint8_t *p = src + (size_t)y * step + (size_t)x * cn;
    const int g = cn == 1 ? p[0] : (p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + (1 << 14)) >> 15;
    char *row = static_cast<char *>(dst) + (size_t)y * dstep;
    if (to_f32)
        reinterpret_cast<float *>(row)[x] = (float)(1.0 / 255.0) * (float)g;
    else
        reinterpret_cast<uint8_t *>(row)[x] = (uint8_t)g;
}

// ------------------------------------------------------------------------------------------------ per processed frame
// win[k] = frames[frame_slot[k]]; rel[4k + {0,1,2,3}] = (relForward.x, relForward.y, relBackward.x, relBackward.y)
__global__ void k_sr_window(SrGeom g, SrWindow w, const float *frames, const float *fwd, const float *bwd, float *win,
                            float *rel) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= g.lr_cols || y >= g.lr_rows) return;
    for (int k = 0; k < w.K; ++k)
        for (int c = 0; c < g.cn; ++c)
            win[k * g.lr_frame + (size_t)y * g.lpc + x * g.cn + c] =
                frames[w.frame_slot[k] * g.lr_frame + (size_t)y * g.lpc + x * g.cn + c];
    const size_t o = (size_t)y * g.lp + x;
    auto F = [&](int slot, int comp) { return fwd[(2 * slot + comp) * g.lr_plane + o]; };
    auto B = [&](int slot, int comp) { return bwd[(2 * slot + comp) * g.lr_plane + o]; };
    auto R = [&](int k, int comp) -> float & { return rel[(4 * k + comp) * g.lr_plane + o]; };
    for (int comp = 0; comp < 4; ++comp) R(w.base, comp) = 0.0f;
    for (int i = w.base - 1; i >= 0; --i)
        for (int comp = 0; comp < 2; ++comp) {
            R(i, comp) = R(i + 1, comp) + F(w.fwd_slot[i], comp);
            R(i, 2 + comp) = R(i + 1, 2 + comp) + B(w.bwd_slot[i + 1], comp);
        }
    for (int i = w.base + 1; i < w.K; ++i)
        for (int comp = 0; comp < 2; ++comp) {
            R(i, comp) = R(i - 1, comp) + B(w.bwd_slot[i], comp);
            R(i, 2 + comp) = R(i - 1, 2 + comp) + F(w.fwd_slot[i - 1], comp);
        }
}

// cuda::resize(INTER_CUBIC) at high-resolution pixel (hy, hx): top-left aligned samples at p * float(1 / scale), taps
// ceil(c - 2) .. floor(c + 2) with replicated borders, normalised by the weight sum.  Accumulates n planes.
template <int N>
__device__ __forceinline__ void cubic_sample(const SrGeom &g, float inv, int hy, int hx, const float *const *src,
                                             const size_t *pitch, const int *chan, float *out) {
    const float xc = (float)hx * inv, yc = (float)hy * inv;
    const float xmin = ceilf(xc - 2.0f), xmax = floorf(xc + 2.0f);
    const float ymin = ceilf(yc - 2.0f), ymax = floorf(yc + 2.0f);
    float sum[N];
#pragma unroll
    for (int i = 0; i < N; ++i) sum[i] = 0.0f;
    float wsum = 0.0f;
    for (float cy = ymin; cy <= ymax; cy += 1.0f) {
        const int iy = min(max(__float2int_rd(cy), 0), g.lr_rows - 1);
        for (float cx = xmin; cx <= xmax; cx += 1.0f) {
            const int ix = min(max(__float2int_rd(cx), 0), g.lr_cols - 1);
            const float wgt = cubic_coeff(xc - cx) * cubic_coeff(yc - cy);
#pragma unroll
            for (int i = 0; i < N; ++i) sum[i] = sum[i] + wgt * src[i][(size_t)iy * pitch[i] + (size_t)ix * chan[i]];
            wsum += wgt;
        }
    }
#pragma unroll
    for (int i = 0; i < N; ++i) out[i] = wsum == 0.0f ? 0.0f : sum[i] / wsum;
}

__global__ void k_sr_maps(SrGeom g, int K, int base, float inv, const float *win, const float *rel, int *idx_fwd,
                          int *idx_bwd, float *hr) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= g.hr_cols || y >= g.hr_rows) return;
    const float s = (float)g.scale;
    for (int k = 0; k < K; ++k) {
        const float *src[4];
        size_t pitch[4];
        int chan[4];
        for (int i = 0; i < 4; ++i) {
            src[i] = rel + (4 * k + i) * g.lr_plane;
            pitch[i] = g.lp;
            chan[i] = 1;
        }
        float m[4];
        cubic_sample<4>(g, inv, y, x, src, pitch, chan, m);
        const float fx = m[0] * s, fy = m[1] * s, bx = m[2] * s, by = m[3] * s;
        // forwardMap = p + backwardMotion, backwardMap = p + forwardMotion (btv_l1_gpu.cu:73-95)
        const int fwd = nearest_index((float)y + by, g.hr_rows) * g.hr_cols + nearest_index((float)x + bx, g.hr_cols);
        const int bwd = nearest_index((float)y + fy, g.hr_rows) * g.hr_cols + nearest_index((float)x + fx, g.hr_cols);
        idx_fwd[k * g.hr_index + (size_t)y * g.hp + x] = fwd;
        idx_bwd[k * g.hr_index + (size_t)y * g.hp + x] = bwd;
    }
    const float *src[4];
    size_t pitch[4];
    int chan[4];
    for (int c = 0; c < 4; ++c) {
        src[c] = win + base * g.lr_frame + min(c, g.cn - 1);
        pitch[c] = g.lpc;
        chan[c] = g.cn;
    }
    float v[4];
    cubic_sample<4>(g, inv, y, x, src, pitch, chan, v);
    for (int c = 0; c < g.cn; ++c) hr[(size_t)y * g.hpc + x * g.cn + c] = v[c];
}

// ------------------------------------------------------------------------------------------------ per iteration
// For low-resolution pixel (y, x) of frame k: b = blur(remap(hr, backwardMap_k)) at (y s, x s), row pass then column pass
// (cudafilters' separable filter, reflect-101), then sign(src_k - b) per channel.
__global__ void k_sr_forward(SrGeom g, SrIter P, const float *hr, const int *idx_bwd, const float *win, int8_t *sign) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, k = blockIdx.z;
    if (x >= g.lr_cols || y >= g.lr_rows) return;
    const int Y = y * g.scale, X = x * g.scale;
    const int *idx = idx_bwd + k * g.hr_index;
    float b[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int j = 0; j < P.bk; ++j) {
        const int r = reflect101(Y - P.anchor + j, g.hr_rows);
        float row[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        for (int i = 0; i < P.bk; ++i) {
            const int cidx = reflect101(X - P.anchor + i, g.hr_cols);
            const float *a = hr + (size_t)__ldg(idx + (size_t)r * g.hp + cidx) * g.cn;
            for (int c = 0; c < g.cn; ++c) row[c] = row[c] + a[c] * P.blur[i];
        }
        for (int c = 0; c < g.cn; ++c) b[c] = b[c] + row[c] * P.blur[j];
    }
    const float *src = win + k * g.lr_frame + (size_t)y * g.lpc + x * g.cn;
    int8_t *out = sign + k * g.sign_plane + (size_t)y * g.sp + x * g.cn;
    for (int c = 0; c < g.cn; ++c) out[c] = (int8_t)diff_sign(src[c], b[c]);
}

// Blur of the sign image upscaled with zeros (non-zero only at multiples of `scale`) at high-resolution pixel (qy, qx):
// the dense filter's row-then-column sums with the zero taps left out (they add exactly zero).
__device__ __forceinline__ void blur_upscaled(const SrGeom &g, const SrIter &P, const int8_t *sign, int qy, int qx, float *out) {
    for (int c = 0; c < 4; ++c) out[c] = 0.0f;
    for (int j = 0; j < P.bk; ++j) {
        const int r = reflect101(qy - P.anchor + j, g.hr_rows);
        if (r % g.scale) continue;
        const int8_t *srow = sign + (size_t)(r / g.scale) * g.sp;
        float row[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        bool any = false;
        for (int i = 0; i < P.bk; ++i) {
            const int cidx = reflect101(qx - P.anchor + i, g.hr_cols);
            if (cidx % g.scale) continue;
            const int8_t *sv = srow + (cidx / g.scale) * g.cn;
            for (int c = 0; c < g.cn; ++c)
                if (sv[c]) {
                    row[c] = row[c] + (float)sv[c] * P.blur[i];
                    any = true;
                }
        }
        if (any)
            for (int c = 0; c < g.cn; ++c)
                if (row[c] != 0.0f) out[c] = out[c] + row[c] * P.blur[j];
    }
}

__global__ void k_sr_update(SrGeom g, SrIter P, const float *hr, const int *idx_fwd, const int8_t *sign, float *dst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= g.hr_cols || y >= g.hr_rows) return;
    const float *p = hr + (size_t)y * g.hpc + x * g.cn;
    float v[4];
    for (int c = 0; c < g.cn; ++c) v[c] = p[c];
    if (P.reg) {
        // calcBtvRegularizationKernel (btv_l1_gpu.cu:192-214): interior pixels only, 0 elsewhere; the float4 diffSign
        // zeroes .w, so a 4th channel gets no regularisation
        float reg[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        const int ks = P.ks;
        if (y >= ks && y < g.hr_rows - ks && x >= ks && x < g.hr_cols - ks) {
            const int creg = g.cn == 4 ? 3 : g.cn;
            for (int m = 0, count = 0; m <= ks; ++m)
                for (int l = ks; l + m >= 0; --l, ++count) {
                    const float *a = hr + (size_t)(y + m) * g.hpc + (x + l) * g.cn;
                    const float *b = hr + (size_t)(y - m) * g.hpc + (x - l) * g.cn;
                    for (int c = 0; c < creg; ++c)
                        reg[c] = reg[c] + P.btv[count] * (diff_sign(v[c], a[c]) - diff_sign(b[c], v[c]));
                }
        }
        // addWeighted(hr, 1, reg, -tau lambda, 0)
        for (int c = 0; c < g.cn; ++c) v[c] = v[c] * 1.0f + reg[c] * P.reg_beta + 0.0f;
    }
    for (int k = 0; k < P.K; ++k) {
        const int q = __ldg(idx_fwd + k * g.hr_index + (size_t)y * g.hp + x);
        float d[4];
        blur_upscaled(g, P, sign + k * g.sign_plane, q / g.hr_cols, q % g.hr_cols, d);
        // addWeighted(hr, 1, diffTerm_k, tau, 0)
        for (int c = 0; c < g.cn; ++c) v[c] = v[c] * 1.0f + d[c] * P.tau + 0.0f;
    }
    float *o = dst + (size_t)y * g.hpc + x * g.cn;
    for (int c = 0; c < g.cn; ++c) o[c] = v[c];
}

// ------------------------------------------------------------------------------------------------ output
// crop by btvKernelSize on every side, then convertTo(CV_8U) (round half to even, saturate) or a float copy
__global__ void k_sr_output(SrGeom g, const float *hr, int crop, int rows, int cols, void *dst, size_t dstep, int to_u8) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols * g.cn || y >= rows) return;
    const float v = hr[(size_t)(y + crop) * g.hpc + crop * g.cn + x];
    char *row = static_cast<char *>(dst) + (size_t)y * dstep;
    if (to_u8)
        reinterpret_cast<uint8_t *>(row)[x] = (uint8_t)min(max(__float2int_rn(v), 0), 255);
    else
        reinterpret_cast<float *>(row)[x] = v;
}

}  // namespace

// getGaussianKernel(n, sigma, CV_32F): OpenCV's bit-exact rule (fixed tables for n <= 9 at sigma <= 0), in double
void sr_gaussian_kernel(int n, double sigma, float *out) {
    static const double t1[] = {1.0}, t3[] = {0.25, 0.5, 0.25}, t5[] = {0.0625, 0.25, 0.375, 0.25, 0.0625},
                        t7[] = {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125},
                        t9[] = {4 / 256.0, 13 / 256.0, 30 / 256.0, 51 / 256.0, 60 / 256.0, 51 / 256.0, 30 / 256.0, 13 / 256.0,
                                4 / 256.0};
    const double *tab = n == 1 ? t1 : n == 3 ? t3 : n == 5 ? t5 : n == 7 ? t7 : n == 9 ? t9 : nullptr;
    if (tab && sigma <= 0) {
        for (int i = 0; i < n; ++i) out[i] = (float)tab[i];
        return;
    }
    const double sx = sigma > 0 ? sigma : std::fma((double)n, 0.15, 0.35);
    const double scale2 = -0.125 / (sx * sx);
    const int h = (n - 1) / 2;
    std::vector<double> v(h + 1);
    double sum = 0;
    for (int i = 0, x = 1 - n; i < h; ++i, x += 2) {
        v[i] = std::exp((double)(x * x) * scale2);
        sum += v[i];
    }
    sum *= 2;
    sum += 1;
    if ((n & 1) == 0) sum += 1;
    const double mul = 1.0 / sum;
    for (int i = 0; i < h; ++i) out[i] = out[n - 1 - i] = (float)(v[i] * mul);
    out[h] = (float)(1.0 * mul);
    if ((n & 1) == 0) out[h + 1] = out[h];
}

}  // namespace b2f

// ================================================================================================ the handle
struct b2f_superres : b2f_handle {
    b2f_superres_params P;
    b2f_handle *flow = nullptr;  // borrowed; NULL: the caller pushes flows

    // the stream: geometry and ring length latched by its first frame
    bool started = false, init_done = false, eos = false, read_done = false;
    int init_reads = 0, store_pos = -1, proc_pos = 0, out_pos = -1;
    int R = 0, L = 1, type = -1;
    b2f::SrGeom g{};
    float *frames = nullptr, *fwd = nullptr, *bwd = nullptr, *win = nullptr, *rel = nullptr, *hr0 = nullptr, *hr1 = nullptr,
          *outs = nullptr;
    int *idx_fwd = nullptr, *idx_bwd = nullptr;
    int8_t *sign = nullptr;
    uint8_t *gray[2] = {nullptr, nullptr};  // work-type frames of the flow wrapper: previous, current
    int gray_cur = 0;
    size_t gray_step = 0;
    std::vector<int> out_crop;  // btvKernelSize each output slot was processed with

    struct Key {
        const void *base = nullptr;
        int lr_rows = 0, lr_cols = 0, cn = 0, scale = 0, L = 0;
        int K = 0, iterations = 0, bk = 0, btv = 0, reg = 0;
        double sigma = 0, alpha = 0, tau = 0, lambda = 0;
        bool operator==(const Key &o) const {
            return base == o.base && lr_rows == o.lr_rows && lr_cols == o.lr_cols && cn == o.cn && scale == o.scale &&
                   L == o.L && K == o.K && iterations == o.iterations && bk == o.bk && btv == o.btv && reg == o.reg && sigma == o.sigma && alpha == o.alpha && tau == o.tau && lambda == o.lambda;
        }
    };
    b2f::GraphCache<Key> graph;

    explicit b2f_superres(const b2f_superres_params &p) : P(p) {}
    int calc(const b2f_image *, const b2f_image *, b2f_image *, cudaStream_t) override { return B2F_BAD_ARG; }
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    const char *default_name() const override { return "SuperResolution.BTVL1_CUDA"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"sr_forward", "sr_update", "sr_maps", "sr_window", "sr_ingest", "sr_output"};
        return cls >= 0 && cls < 6 ? n[cls] : "";
    }
    size_t workspace_bytes(int, int, int) override { return arena.capacity(); }

    int validate() const;
    void reset_stream() {
        started = init_done = eos = read_done = false;
        init_reads = 0;
        store_pos = -1;
        proc_pos = 0;
        out_pos = -1;
        type = -1;
    }
    int radius() const { return started ? R : P.temporal_area_radius; }
    // btvKernelSize of the output the next pop returns: the slot's, unless that pop's processFrame overwrites the slot
    // first (R = 0: a ring of one, where the reference returns the frame processed in the same call)
    int next_crop() const {
        const int next = out_pos + 1;
        const bool overwritten = proc_pos < store_pos && (proc_pos + 1) % L == next % L;
        return overwritten ? P.btv_kernel_size : out_crop[next % L];
    }
    bool wants_frame() const {
        if (!init_done) return !eos && init_reads < 2 * radius() + 1;
        return !eos && !read_done && out_pos < store_pos;
    }
    int start(const b2f_image *frame, cudaStream_t s);
    int read(const b2f_image *frame, const b2f_image *const *flows, cudaStream_t s);
    int process(int idx, cudaStream_t s);
    int after_read(cudaStream_t s);
    int pop(b2f_image *out, int *produced, cudaStream_t s);
};

int b2f_superres::set_param(int id, double v) {
    switch (id) {
        case B2F_SR_SCALE: P.scale = static_cast<int>(v); return B2F_OK;
        case B2F_SR_ITERATIONS: P.iterations = static_cast<int>(v); return B2F_OK;
        case B2F_SR_TAU: P.tau = v; return B2F_OK;
        case B2F_SR_LAMBDA: P.lambda = v; return B2F_OK;
        case B2F_SR_ALPHA: P.alpha = v; return B2F_OK;
        case B2F_SR_BTV_KERNEL_SIZE: P.btv_kernel_size = static_cast<int>(v); return B2F_OK;
        case B2F_SR_BLUR_KERNEL_SIZE: P.blur_kernel_size = static_cast<int>(v); return B2F_OK;
        case B2F_SR_BLUR_SIGMA: P.blur_sigma = v; return B2F_OK;
        case B2F_SR_TEMPORAL_AREA_RADIUS: P.temporal_area_radius = static_cast<int>(v); return B2F_OK;
        default: return B2F_BAD_ARG;
    }
}

int b2f_superres::get_param(int id, double *v) const {
    switch (id) {
        case B2F_SR_SCALE: *v = P.scale; return B2F_OK;
        case B2F_SR_ITERATIONS: *v = P.iterations; return B2F_OK;
        case B2F_SR_TAU: *v = P.tau; return B2F_OK;
        case B2F_SR_LAMBDA: *v = P.lambda; return B2F_OK;
        case B2F_SR_ALPHA: *v = P.alpha; return B2F_OK;
        case B2F_SR_BTV_KERNEL_SIZE: *v = P.btv_kernel_size; return B2F_OK;
        case B2F_SR_BLUR_KERNEL_SIZE: *v = P.blur_kernel_size; return B2F_OK;
        case B2F_SR_BLUR_SIGMA: *v = P.blur_sigma; return B2F_OK;
        case B2F_SR_TEMPORAL_AREA_RADIUS: *v = P.temporal_area_radius; return B2F_OK;
        default: return B2F_BAD_ARG;
    }
}

// btv_l1_cuda.cpp:310-316, plus cudafilters' odd blur size of at most 32 (filtering.cpp:441-442, 568) and this engine's
// radius limit
int b2f_superres::validate() const {
    const b2f_superres_params &p = P;
    if (!(p.scale > 1) || !(p.iterations > 0) || !(p.tau > 0) || !(p.alpha > 0)) return B2F_BAD_ARG;
    if (!(p.btv_kernel_size > 0 && p.btv_kernel_size <= 16)) return B2F_BAD_ARG;
    if (!(p.blur_kernel_size > 0) || !(p.blur_sigma >= 0) || (p.blur_kernel_size & 1) == 0 || p.blur_kernel_size > 32)
        return B2F_BAD_ARG;
    if (p.temporal_area_radius < 0 || p.temporal_area_radius > B2F_SR_MAX_RADIUS) return B2F_BAD_ARG;
    if (started && (g.hr_rows <= 2 * p.btv_kernel_size || g.hr_cols <= 2 * p.btv_kernel_size)) return B2F_BAD_ARG;
    return B2F_OK;
}

static bool frame_ok(const b2f_image *f) {
    return f && f->data && f->rows > 0 && f->cols > 0 &&
           (f->type == B2F_8UC1 || f->type == B2F_8UC3 || f->type == B2F_8UC4);
}
static int channels_of(int type) { return type == B2F_8UC1 ? 1 : type == B2F_8UC3 ? 3 : 4; }

static int gray_to_f32(const b2f_handle *h) { return h->algo == b2f::ALGO_BROX ? 1 : 0; }

int b2f_superres::start(const b2f_image *frame, cudaStream_t s) {
    using namespace b2f;
    R = P.temporal_area_radius;
    L = 2 * R + 1;
    SrGeom n{};
    n.lr_rows = frame->rows;
    n.lr_cols = frame->cols;
    n.cn = channels_of(frame->type);
    n.scale = P.scale;
    n.hr_rows = frame->rows * P.scale;
    n.hr_cols = frame->cols * P.scale;
    if (n.hr_rows <= 2 * P.btv_kernel_size || n.hr_cols <= 2 * P.btv_kernel_size) return B2F_BAD_ARG;
    if ((double)n.hr_rows * n.hr_cols * 4 > 2147483647.0) return B2F_BAD_ARG;  // int32 linear indices
    n.lp = round_up(n.lr_cols, 32);
    n.lpc = round_up(n.lr_cols * n.cn, 32);
    n.hpc = n.hr_cols * n.cn;
    n.hp = round_up(n.hr_cols, 32);
    n.sp = round_up(n.lr_cols * n.cn, 128);
    n.lr_plane = (size_t)n.lp * n.lr_rows;
    n.lr_frame = (size_t)n.lpc * n.lr_rows;
    n.hr_image = (size_t)n.hpc * n.hr_rows;
    n.hr_index = (size_t)n.hp * n.hr_rows;
    n.sign_plane = (size_t)n.sp * n.lr_rows;
    gray_step = (size_t)round_up(n.lr_cols * 4, 256);
    for (int pass = 0; pass < 2; ++pass) {
        arena.begin(pass == 0);
        frames = static_cast<float *>(arena.bytes(4 * n.lr_frame * L));
        fwd = static_cast<float *>(arena.bytes(4 * n.lr_plane * 2 * L));
        bwd = static_cast<float *>(arena.bytes(4 * n.lr_plane * 2 * L));
        win = static_cast<float *>(arena.bytes(4 * n.lr_frame * L));
        rel = static_cast<float *>(arena.bytes(4 * n.lr_plane * 4 * L));
        hr0 = static_cast<float *>(arena.bytes(4 * n.hr_image));
        hr1 = static_cast<float *>(arena.bytes(4 * n.hr_image));
        outs = static_cast<float *>(arena.bytes(4 * n.hr_image * L));
        idx_fwd = static_cast<int *>(arena.bytes(4 * n.hr_index * L));
        idx_bwd = static_cast<int *>(arena.bytes(4 * n.hr_index * L));
        sign = static_cast<int8_t *>(arena.bytes(n.sign_plane * L));
        gray[0] = static_cast<uint8_t *>(arena.bytes(gray_step * n.lr_rows));
        gray[1] = static_cast<uint8_t *>(arena.bytes(gray_step * n.lr_rows));
        if (pass == 0) {
            cudaError_t e = arena.reserve(arena.used());
            if (e != cudaSuccess) {
                last_cuda_error = e;
                cudaGetLastError();
                return B2F_OUT_OF_MEMORY;
            }
        }
    }
    (void)s;
    g = n;
    type = frame->type;
    out_crop.assign(L, 0);
    started = true;
    return B2F_OK;
}

// readNextFrame (btv_l1_cuda.cpp:532-553): store the frame, then flows (prev -> cur) into forward at(pos - 1) and
// (cur -> prev) into backward at(pos)
int b2f_superres::read(const b2f_image *frame, const b2f_image *const *flows, cudaStream_t s) {
    using namespace b2f;
    if (!frame) {
        eos = true;
        return after_read(s);
    }
    if (!started) {
        int st = start(frame, s);
        if (st != B2F_OK) return st;
    } else {
        if (frame->type != type) return B2F_UNSUPPORTED_TYPE;
        if (frame->rows != g.lr_rows || frame->cols != g.lr_cols) return B2F_SIZE_MISMATCH;
    }
    if (frame->step < (size_t)frame->cols * g.cn) return B2F_BAD_ARG;
    if (flows && store_pos >= 0) {
        for (int i = 0; i < 4; ++i) {
            const b2f_image *f = flows[i];
            if (!f || !f->data) return B2F_BAD_ARG;
            if (f->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
            if (f->rows != g.lr_rows || f->cols != g.lr_cols) return B2F_SIZE_MISMATCH;
            if (f->step < (size_t)f->cols * 4) return B2F_BAD_ARG;
        }
    }
    const int pos = store_pos + 1;
    Ctx c = make_ctx(s);
    const dim3 blk(32, 8);
    B2F_LAUNCH(c, CLS_INGEST, (double)g.lr_rows * g.lr_cols * g.cn * 5, k_sr_ingest, dim3(div_up(g.lr_cols * g.cn, 32), div_up(g.lr_rows, 8)),
               blk, 0, static_cast<const uint8_t *>(frame->data), frame->step, g.lr_rows, g.lr_cols, g.cn,
               frames + (size_t)(pos % L) * g.lr_frame, g.lpc);
    const int fslot = (pos - 1 + L) % L, bslot = pos % L;
    if (pos > 0 && flows) {
        float *dst[4] = {fwd + 2 * fslot * g.lr_plane, fwd + (2 * fslot + 1) * g.lr_plane, bwd + 2 * bslot * g.lr_plane,
                         bwd + (2 * bslot + 1) * g.lr_plane};
        for (int i = 0; i < 4; ++i)
            c.check(cudaMemcpy2DAsync(dst[i], (size_t)g.lp * 4, flows[i]->data, flows[i]->step, (size_t)g.lr_cols * 4,
                                      g.lr_rows, cudaMemcpyDeviceToDevice, s));
    }
    if (!flows) {
        // the wrapper's conversion of the raw frame to the flow engine's work type
        const int f32 = gray_to_f32(flow);
        const int cur = gray_cur ^ 1;
        B2F_LAUNCH(c, CLS_INGEST, (double)g.lr_rows * g.lr_cols * (g.cn + 4), k_sr_gray, dim3(div_up(g.lr_cols, 32), div_up(g.lr_rows, 8)),
                   blk, 0, static_cast<const uint8_t *>(frame->data), frame->step, g.lr_rows, g.lr_cols, g.cn, gray[cur],
                   gray_step, f32);
        if (!c.ok()) return finish(c, s);
        if (pos > 0) {
            const int wt = f32 ? B2F_32FC1 : B2F_8UC1;
            b2f_image prev{gray[gray_cur], gray_step, g.lr_rows, g.lr_cols, wt}, now{gray[cur], gray_step, g.lr_rows, g.lr_cols, wt};
            b2f_image u{fwd + 2 * fslot * g.lr_plane, (size_t)g.lp * 4, g.lr_rows, g.lr_cols, B2F_32FC1};
            b2f_image v{fwd + (2 * fslot + 1) * g.lr_plane, (size_t)g.lp * 4, g.lr_rows, g.lr_cols, B2F_32FC1};
            b2f_image bu{bwd + 2 * bslot * g.lr_plane, (size_t)g.lp * 4, g.lr_rows, g.lr_cols, B2F_32FC1};
            b2f_image bv{bwd + (2 * bslot + 1) * g.lr_plane, (size_t)g.lp * 4, g.lr_rows, g.lr_cols, B2F_32FC1};
            int st = b2f_calc_uv(flow, &prev, &now, &u, &v, s);
            if (st == B2F_OK) st = b2f_calc_uv(flow, &now, &prev, &bu, &bv, s);
            if (st != B2F_OK) {
                last_cuda_error = b2f_last_cuda_error(flow);
                return st;
            }
        }
        gray_cur = cur;
    }
    int st = finish(c, s);
    if (st != B2F_OK) return st;
    store_pos = pos;
    if (!init_done) ++init_reads;
    else read_done = true;
    return after_read(s);
}

// initImpl's processFrame(0 .. R) once its 2R + 1 reads are done (frames past the end of a short stream are skipped)
int b2f_superres::after_read(cudaStream_t s) {
    if (init_done || (init_reads < 2 * radius() + 1 && !eos)) return B2F_OK;
    if (started)
        for (int i = 0; i <= R && i <= store_pos; ++i) {
            int st = process(i, s);
            if (st != B2F_OK) return st;
        }
    proc_pos = R;
    out_pos = -1;
    init_done = true;
    return B2F_OK;
}

int b2f_superres::process(int idx, cudaStream_t s) {
    using namespace b2f;
    const int start_i = idx - R > 0 ? idx - R : 0;
    const int end_i = start_i + 2 * R < store_pos ? start_i + 2 * R : store_pos;
    SrWindow w{};
    w.K = end_i - start_i + 1;
    w.base = idx - start_i;
    for (int i = start_i, k = 0; i <= end_i; ++i, ++k) {
        w.frame_slot[k] = i % L;
        w.fwd_slot[k] = i < end_i ? i % L : 0;
        w.bwd_slot[k] = i > start_i ? i % L : 0;
    }
    SrIter it{};
    it.bk = P.blur_kernel_size;
    it.anchor = it.bk / 2;
    sr_gaussian_kernel(it.bk, P.blur_sigma, it.blur);
    it.ks = (P.btv_kernel_size - 1) / 2;
    {
        const float af = static_cast<float>(P.alpha);
        for (int m = 0, ind = 0; m <= it.ks; ++m)
            for (int l = it.ks; l + m >= 0; --l, ++ind) it.btv[ind] = static_cast<float>(std::pow((double)af, std::abs(m) + std::abs(l)));
    }
    it.K = w.K;
    it.reg = P.lambda > 0;
    it.reg_beta = static_cast<float>(-P.tau * P.lambda);
    it.tau = static_cast<float>(P.tau);
    const float inv = static_cast<float>(1.0 / g.scale);  // the stream's latched scale

    Ctx c = make_ctx(s);
    const dim3 blk(32, 8);
    const dim3 glr(div_up(g.lr_cols, 32), div_up(g.lr_rows, 8)), ghr(div_up(g.hr_cols, 32), div_up(g.hr_rows, 8));
    const double lr_px = (double)g.lr_rows * g.lr_cols, hr_px = (double)g.hr_rows * g.hr_cols;
    B2F_LAUNCH(c, CLS_WINDOW, lr_px * w.K * (8.0 * g.cn + 32), k_sr_window, glr, blk, 0, g, w, frames, fwd, bwd, win, rel);
    B2F_LAUNCH(c, CLS_MAPS, lr_px * (w.K * 16.0 + 4 * g.cn) + hr_px * (w.K * 8.0 + 4 * g.cn), k_sr_maps, ghr, blk, 0, g, w.K,
               w.base, inv, win, rel, idx_fwd, idx_bwd, hr0);
    const int iters = P.iterations;
    const double fwd_bytes = lr_px * w.K * (4.0 * g.cn + g.cn) + hr_px * w.K * 4.0 * it.bk * it.bk / (g.scale * g.scale) +
                             hr_px * 4.0 * g.cn;
    const double upd_bytes = hr_px * (8.0 * g.cn + 4.0 * w.K) + lr_px * w.K * g.cn;
    auto body = [&](Ctx &cc) {
        float *a = hr0, *b = hr1;
        for (int i = 0; i < iters; ++i) {
            B2F_LAUNCH(cc, CLS_ITER_FORWARD, fwd_bytes, k_sr_forward, dim3(glr.x, glr.y, w.K), blk, 0, g, it, a, idx_bwd, win, sign);
            B2F_LAUNCH(cc, CLS_ITER_UPDATE, upd_bytes, k_sr_update, ghr, blk, 0, g, it, a, idx_fwd, sign, b);
            float *t = a;
            a = b;
            b = t;
        }
        if (cc.stats) cc.stats->iterations_run = iters;
    };
    Key key;
    key.base = arena.capacity() ? static_cast<const void *>(frames) : nullptr;
    key.lr_rows = g.lr_rows;
    key.lr_cols = g.lr_cols;
    key.cn = g.cn;
    key.scale = g.scale;
    key.L = L;
    key.K = w.K;
    key.iterations = iters;
    key.bk = it.bk;
    key.btv = P.btv_kernel_size;
    key.reg = it.reg;
    key.sigma = P.blur_sigma;
    key.alpha = P.alpha;
    key.tau = P.tau;
    key.lambda = P.lambda;
    if (!(knobs.use_graph && !profiling && graph.run(*this, c, s, key, body))) {
        if (c.ok()) body(c);
    }
    const float *result = (iters & 1) ? hr1 : hr0;
    c.check(cudaMemcpyAsync(outs + (size_t)(idx % L) * g.hr_image, result, 4 * g.hr_image, cudaMemcpyDeviceToDevice, s));
    out_crop[idx % L] = P.btv_kernel_size;
    stats.calls++;
    return finish(c, s);
}

int b2f_superres::pop(b2f_image *out, int *produced, cudaStream_t s) {
    using namespace b2f;
    *produced = 0;
    if (!init_done || wants_frame()) return B2F_BAD_ARG;  // push the frame the schedule reads next first
    if (out_pos >= store_pos) return B2F_OK;              // end of the stream
    if (!out || !out->data) return B2F_BAD_ARG;
    const int want_u8 = out->type == type, want_f32 = out->type == (type == B2F_8UC1 ? B2F_32FC1 : type == B2F_8UC3 ? B2F_32FC3 : B2F_32FC4);
    if (!want_u8 && !want_f32) return B2F_UNSUPPORTED_TYPE;
    const int next = out_pos + 1;
    const int crop = next_crop();
    const int rows = g.hr_rows - 2 * crop, cols = g.hr_cols - 2 * crop;
    if (out->rows != rows || out->cols != cols) return B2F_SIZE_MISMATCH;
    if (out->step < (size_t)cols * g.cn * (want_u8 ? 1 : 4)) return B2F_BAD_ARG;
    int st;
    if (proc_pos < store_pos) {
        st = process(proc_pos + 1, s);
        if (st != B2F_OK) return st;
        ++proc_pos;
    }
    Ctx c = make_ctx(s);
    B2F_LAUNCH(c, CLS_OUTPUT, (double)rows * cols * g.cn * (want_u8 ? 5 : 8), k_sr_output,
               dim3(div_up(cols * g.cn, 32), div_up(rows, 8)), dim3(32, 8), 0, g, outs + (size_t)(next % L) * g.hr_image, crop,
               rows, cols, out->data, out->step, want_u8);
    st = finish(c, s);
    if (st != B2F_OK) return st;
    out_pos = next;
    read_done = false;
    *produced = 1;
    return B2F_OK;
}

// ================================================================================================ C ABI
extern "C" {

void b2f_superres_default_params(b2f_superres_params *p) {
    if (!p) return;
    p->scale = 4;
    p->iterations = 180;
    p->tau = 1.3;
    p->lambda = 0.03;
    p->alpha = 0.7;
    p->btv_kernel_size = 7;
    p->blur_kernel_size = 5;
    p->blur_sigma = 0.0;
    p->temporal_area_radius = 4;
}

static bool flow_engine_ok(const b2f_handle *h) {
    return !h || h->algo == b2f::ALGO_TVL1 || h->algo == b2f::ALGO_FARNEBACK || h->algo == b2f::ALGO_BROX ||
           h->algo == b2f::ALGO_DENSELK;
}

int b2f_superres_create(const b2f_superres_params *p, b2f_handle *flow, b2f_superres **out) {
    if (!out) return B2F_BAD_ARG;
    *out = nullptr;
    if (!flow_engine_ok(flow)) return B2F_BAD_ARG;
    b2f_superres_params d;
    b2f_superres_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f_superres(d);
    if (!*out) return B2F_OUT_OF_MEMORY;
    (*out)->flow = flow;
    return B2F_OK;
}

void b2f_superres_destroy(b2f_superres *sr) { delete sr; }

int b2f_superres_set_flow(b2f_superres *sr, b2f_handle *flow) {
    if (!sr || !flow_engine_ok(flow)) return B2F_BAD_ARG;
    sr->flow = flow;
    return B2F_OK;
}

int b2f_superres_set_param(b2f_superres *sr, int id, double value) { return b2f_set_param(sr, id, value); }
int b2f_superres_get_param(const b2f_superres *sr, int id, double *value) { return b2f_get_param(sr, id, value); }

int b2f_superres_wants_frame(const b2f_superres *sr, int *wants) {
    if (!sr || !wants) return B2F_BAD_ARG;
    *wants = sr->wants_frame() ? 1 : 0;
    return B2F_OK;
}

static int sr_push(b2f_superres *sr, const b2f_image *frame, const b2f_image *const *flows, void *cuda_stream) {
    if (!sr) return B2F_BAD_ARG;
    int st = sr->validate();
    if (st != B2F_OK) return st;
    if (!frame) {
        if (sr->eos) return B2F_OK;
        return sr->read(nullptr, nullptr, static_cast<cudaStream_t>(cuda_stream));
    }
    if (!frame->data || frame->rows <= 0 || frame->cols <= 0) return B2F_BAD_ARG;
    if (!frame_ok(frame)) return B2F_UNSUPPORTED_TYPE;
    if (!sr->wants_frame()) return B2F_BAD_ARG;
    if (!flows && !sr->flow) return B2F_BAD_ARG;
    if (flows && sr->flow) return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    b2f::DeviceScope dev(frame->data, s);
    if (!sr->bind_device()) return B2F_BAD_ARG;
    return sr->read(frame, flows, s);
}

int b2f_superres_push(b2f_superres *sr, const b2f_image *frame, void *cuda_stream) {
    return sr_push(sr, frame, nullptr, cuda_stream);
}

int b2f_superres_push_flows(b2f_superres *sr, const b2f_image *frame, const b2f_image *fwd_u, const b2f_image *fwd_v,
                            const b2f_image *bwd_u, const b2f_image *bwd_v, void *cuda_stream) {
    const b2f_image *f[4] = {fwd_u, fwd_v, bwd_u, bwd_v};
    return sr_push(sr, frame, f, cuda_stream);
}

int b2f_superres_pop(b2f_superres *sr, b2f_image *out, int *produced, void *cuda_stream) {
    if (!sr || !produced) return B2F_BAD_ARG;
    *produced = 0;
    int st = sr->validate();
    if (st != B2F_OK) return st;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    b2f::DeviceScope dev(out ? out->data : nullptr, s);
    if (!sr->bind_device()) return B2F_BAD_ARG;
    return sr->pop(out, produced, s);
}

int b2f_superres_output_size(const b2f_superres *sr, int *rows, int *cols) {
    if (!sr || !rows || !cols || !sr->started) return B2F_BAD_ARG;
    // the next output's crop once it has been processed, else the current btvKernelSize
    const bool ready = sr->init_done && sr->out_pos < sr->store_pos;
    const int crop = ready ? sr->next_crop() : sr->P.btv_kernel_size;
    *rows = sr->g.hr_rows - 2 * crop;
    *cols = sr->g.hr_cols - 2 * crop;
    return B2F_OK;
}

int b2f_superres_reset(b2f_superres *sr) {
    if (!sr) return B2F_BAD_ARG;
    sr->reset_stream();
    return B2F_OK;
}

int b2f_superres_collect_garbage(b2f_superres *sr) {
    if (!sr) return B2F_BAD_ARG;
    sr->reset_stream();
    sr->graph.destroy();
    sr->arena.release();
    return B2F_OK;
}

int b2f_superres_get_stats(b2f_superres *sr, b2f_stats *out) { return b2f_get_stats(sr, out); }
int b2f_superres_reset_stats(b2f_superres *sr) { return b2f_reset_stats(sr); }
int b2f_superres_last_cuda_error(const b2f_superres *sr) { return sr ? sr->last_cuda_error : 0; }

// GpuOpticalFlow::calc (superres/src/optical_flow.cpp:456-497): both frames converted to the engine's work type (8UC1 for
// Farneback, DualTVL1 and PyrLK, 32FC1 in [0, 1] for Brox), then calc with planar (flow2 given) or interleaved output
int b2f_calc_ext(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *flow1, b2f_image *flow2,
                 void *cuda_stream) {
    using namespace b2f;
    if (!h || !I0 || !I1 || !flow1 || !I0->data || !I1->data || !flow1->data) return B2F_BAD_ARG;
    if (!flow_engine_ok(h)) return B2F_BAD_ARG;
    if (!frame_ok(I0) || !frame_ok(I1)) return B2F_UNSUPPORTED_TYPE;
    if (I0->type != I1->type) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    const int cn = channels_of(I0->type), f32 = gray_to_f32(h);
    if (I0->step < (size_t)I0->cols * cn || I1->step < (size_t)I1->cols * cn) return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceScope dev(I0->data, s);
    if (!h->bind_device()) return B2F_BAD_ARG;
    b2f_image w0 = *I0, w1 = *I1;
    if (cn != 1 || f32) {
        const size_t step = (size_t)round_up(I0->cols * 4, 256), need = 2 * step * I0->rows;
        if (need > h->ext_stage_bytes) {
            if (h->ext_stage) cudaFree(h->ext_stage);
            h->ext_stage = nullptr;
            h->ext_stage_bytes = 0;
            cudaError_t e = cudaMalloc(&h->ext_stage, need);
            if (e != cudaSuccess) {
                h->last_cuda_error = e;
                cudaGetLastError();
                return B2F_OUT_OF_MEMORY;
            }
            h->ext_stage_bytes = need;
        }
        char *d0 = static_cast<char *>(h->ext_stage), *d1 = d0 + step * I0->rows;
        Ctx c = h->make_ctx(s);
        c.stats = nullptr;  // not the engine's own launches
        const dim3 grid(div_up(I0->cols, 32), div_up(I0->rows, 8)), blk(32, 8);
        B2F_LAUNCH(c, -1, 0, k_sr_gray, grid, blk, 0, static_cast<const uint8_t *>(I0->data), I0->step, I0->rows, I0->cols,
                   cn, d0, step, f32);
        B2F_LAUNCH(c, -1, 0, k_sr_gray, grid, blk, 0, static_cast<const uint8_t *>(I1->data), I1->step, I1->rows, I1->cols,
                   cn, d1, step, f32);
        if (!c.ok()) {
            h->last_cuda_error = c.err;
            cudaGetLastError();
            return B2F_CUDA_ERROR;
        }
        const int wt = f32 ? B2F_32FC1 : B2F_8UC1;
        w0 = b2f_image{d0, step, I0->rows, I0->cols, wt};
        w1 = b2f_image{d1, step, I0->rows, I0->cols, wt};
    }
    return flow2 ? b2f_calc_uv(h, &w0, &w1, flow1, flow2, cuda_stream) : b2f_calc(h, &w0, &w1, flow1, cuda_stream);
}

}  // extern "C"
