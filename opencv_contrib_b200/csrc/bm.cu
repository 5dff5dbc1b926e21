// bm.cu -- cudalegacy's block-matching optical flow: cv::cuda::FastOpticalFlowBM (a dense handle engine) and
// cv::cuda::calcOpticalFlowBM (a free function, one vector per grid cell).  What both compute is stated in numpy by
// oracle/bm_model.py; the engine equals it bit for bit.
//
// FastBM (reference: modules/cudalegacy/src/bm_fast.cpp:62-88, src/cuda/bm_fast.cu:70-290).  The reference pads both
// frames by search_window/2 + block_window/2 with cudev's reflect-101 rule, then walks every pixel of a 128x32 tile one
// after another.  Here one CTA owns a 64-row tile whose columns are one warp wide: both frames' windows are staged in
// shared memory once (the border resolved at load time, so no padded copies), and each warp walks a 16-row strip.  Per
// candidate offset, lane c keeps the vertical sum C_c over block_window rows of column c (slid down the strip), and the
// box sum of output lane l is C_l + ... + C_{l+2br}, taken across lanes with shuffles.  So one warp produces
// 32 - 2br output columns.  The winner is the minimum of (D, rank(k)), rank(k) = tie_pref(k mod 128) * nq + k div 128:
// thread t = k mod 128 of the reference keeps its first strict minimum over k = t, t + 128, ..., and its key-value
// reduction (a halving tree over lanes 16, 8, 4, 2, 1 inside each warp, then over warps 2, 1, the lower position keeping
// ties) prefers the thread whose bits 5, 6, 0, 1, 2, 3, 4 are least, in that order of significance.  The pair is
// packed into one int32 when it cannot overflow, else into an int64 (chosen from the window sizes).
//
// Grid BM (reference: src/bm.cpp:60-202, src/cuda/bm.cu:56-160).  One warp per cell: the spiral candidates are taken 32
// at a time (each lane one, its offset computed in closed form), and the batch's sequential outcome is resolved with a
// ballot for the first accepting lane and warp reductions for the minimum and the tie sums over the lanes before it.
#include "common.cuh"

#include <climits>
#include <new>

namespace b2f {
namespace {

constexpr unsigned FULL = 0xffffffffu;

// cudev BrdReflect101 (cudev/ptr2d/extrapolation.hpp): one fold and a modulo, valid for any i and any len >= 1.
__host__ __device__ __forceinline__ int reflect101_cudev(int i, int len) {
    const int last = len - 1;
    const int hi = abs(last - abs(last - i)) % len;
    return abs(hi) % len;
}

// ------------------------------------------------------------------------------------------- FastBM
constexpr int FBM_WARPS = 4;                   // warps per CTA, stacked vertically
constexpr int FBM_STRIP = 16;                  // output rows per warp
constexpr int FBM_TH = FBM_WARPS * FBM_STRIP;  // tile rows
constexpr int FBM_MAX_SEARCH = 109;            // the reference's shared-memory limit (see b2f_fastbm_params)
constexpr int FBM_MAX_BLOCK = 31;              // one warp must keep at least 2 output columns

struct FbmKeys {
    int bits;  // rank bits
    int nq;    // ceil(sw^2 / 128): rank(k) = tie_pref(k mod 128) * nq + k div 128
    bool wide;
};

// Where thread t's candidate stands among ties after the reference's reduceKeyVal<128>: warp bits reversed (the last
// merge is between warps 0 and 1), then lane bits reversed.  A bit permutation that is its own inverse.
__host__ __device__ __forceinline__ int tie_pref(int t) {
    int p = 0;
    for (int b = 0; b < 5; ++b) p |= ((t >> b) & 1) << (4 - b);
    return p | (((t >> 5) & 1) << 6) | (((t >> 6) & 1) << 5);
}

static FbmKeys fbm_keys(int sw, int bw) {
    FbmKeys k;
    const int n = sw * sw;
    k.nq = (n + 127) / 128;
    int rank_max = 0;
    for (int r = 0; r < 128 && r < n; ++r) {  // the rank of the last k with k mod 128 == r
        const int v = tie_pref(r) * k.nq + (n - 1 - r) / 128;
        if (v > rank_max) rank_max = v;
    }
    k.bits = 0;
    while ((1 << k.bits) <= rank_max) ++k.bits;
    const long long dmax = 255LL * bw * bw;
    k.wide = ((dmax << k.bits) + rank_max) > (long long)INT_MAX;
    return k;
}

// sum of v over lanes [lane, lane + bw) by doubling (lanes that run past 31 read garbage and are not written)
__device__ __forceinline__ int lane_window_sum(int v, int bw) {
    int acc = 0, off = 0, w = v;
    for (int s = 1;; s <<= 1) {
        if (bw & s) {
            acc += __shfl_down_sync(FULL, w, off);
            off += s;
        }
        if ((s << 1) > bw) break;
        w += __shfl_down_sync(FULL, w, s);
    }
    return acc;
}

template <bool WIDE>
struct FbmKey;
template <>
struct FbmKey<false> {
    typedef int T;
    static __device__ __forceinline__ T init() { return INT_MAX; }
    static __device__ __forceinline__ T fold(T best, int d, int bits, int rank) { return __viaddmin_s32(d << bits, rank, best); }
};
template <>
struct FbmKey<true> {
    typedef long long T;
    static __device__ __forceinline__ T init() { return LLONG_MAX; }
    static __device__ __forceinline__ T fold(T best, int d, int bits, int rank) {
        const long long k = ((long long)d << bits) | rank;
        return k < best ? k : best;
    }
};

template <bool WIDE>
__global__ void __launch_bounds__(FBM_WARPS * 32) k_fastbm(const uint8_t *__restrict__ I0, size_t s0,
                                                          const uint8_t *__restrict__ I1, size_t s1, int rows, int cols,
                                                          float *fx, size_t fxs, float *fy, size_t fys, int interleaved,
                                                          int sw, int br, int bits, int nq) {
    typedef FbmKey<WIDE> K;
    extern __shared__ uint8_t sm[];
    const int sr = sw / 2, bw = 2 * br + 1, ow = 32 - 2 * br;
    const int x0 = blockIdx.x * ow, y0 = blockIdx.y * FBM_TH;
    const int h0 = FBM_TH + 2 * br;  // I0 stage: h0 x 32, origin (y0 - br, x0 - br)
    const int w1 = 32 + sw - 1, h1 = h0 + sw - 1;  // I1 stage: h1 x w1, origin (y0 - br - sr, x0 - br - sr)
    uint8_t *a = sm, *b = sm + h0 * 32;
    for (int r = threadIdx.x >> 5; r < h0; r += FBM_WARPS) {
        const uint8_t *src = I0 + (size_t)reflect101_cudev(y0 - br + r, rows) * s0;
        a[r * 32 + (threadIdx.x & 31)] = src[reflect101_cudev(x0 - br + (int)(threadIdx.x & 31), cols)];
    }
    for (int r = threadIdx.x >> 5; r < h1; r += FBM_WARPS) {
        const uint8_t *src = I1 + (size_t)reflect101_cudev(y0 - br - sr + r, rows) * s1;
        for (int c = threadIdx.x & 31; c < w1; c += 32) b[r * w1 + c] = src[reflect101_cudev(x0 - br - sr + c, cols)];
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, ws = (threadIdx.x >> 5) * FBM_STRIP;
    typename K::T best[FBM_STRIP];
#pragma unroll
    for (int s = 0; s < FBM_STRIP; ++s) best[s] = K::init();

    for (int dy = 0; dy < sw; ++dy) {
        for (int dx = 0; dx < sw; ++dx) {
            const int k = dy * sw + dx;
            const int rank = tie_pref(k & 127) * nq + (k >> 7);
            const uint8_t *pa = a + lane, *pb = b + dy * w1 + lane + dx;
            auto d = [&](int q) { return abs((int)pa[q * 32] - (int)pb[q * w1]); };
            int C = 0;
            for (int q = ws; q <= ws + 2 * br; ++q) C += d(q);
#pragma unroll
            for (int s = 0; s < FBM_STRIP; ++s) {
                if (s > 0) C += d(ws + s + 2 * br) - d(ws + s - 1);
                best[s] = K::fold(best[s], lane_window_sum(C, bw), bits, rank);
            }
        }
    }

    const int x = x0 + lane;
    if (lane >= ow || x >= cols) return;
    const typename K::T mask = ((typename K::T)1 << bits) - 1;
#pragma unroll
    for (int s = 0; s < FBM_STRIP; ++s) {
        const int y = y0 + ws + s;
        if (y >= rows) break;
        const int r = (int)(best[s] & mask);
        const int kk = tie_pref(r / nq) + 128 * (r % nq);
        const int ky = kk / sw;
        const float u = (float)(kk - ky * sw - sr), v = (float)(ky - sr);
        if (interleaved) {
            reinterpret_cast<float2 *>(reinterpret_cast<char *>(fx) + (size_t)y * fxs)[x] = make_float2(u, v);
        } else {
            reinterpret_cast<float *>(reinterpret_cast<char *>(fx) + (size_t)y * fxs)[x] = u;
            reinterpret_cast<float *>(reinterpret_cast<char *>(fy) + (size_t)y * fys)[x] = v;
        }
    }
}

class FastBMEngine : public b2f_handle {
public:
    explicit FastBMEngine(const b2f_fastbm_params &p) : P(p) { algo = ALGO_FASTBM; }
    b2f_fastbm_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override {
        switch (id) {
            case B2F_FBM_SEARCH_WINDOW: P.search_window = static_cast<int>(v); return B2F_OK;
            case B2F_FBM_BLOCK_WINDOW: P.block_window = static_cast<int>(v); return B2F_OK;
            default: return B2F_BAD_ARG;
        }
    }
    int get_param(int id, double *v) const override {
        switch (id) {
            case B2F_FBM_SEARCH_WINDOW: *v = P.search_window; return B2F_OK;
            case B2F_FBM_BLOCK_WINDOW: *v = P.block_window; return B2F_OK;
            default: return B2F_BAD_ARG;
        }
    }
    const char *default_name() const override { return "DenseOpticalFlow.FastOpticalFlowBM"; }
    const char *class_name(int cls) const override { return cls == 0 ? "fastbm" : ""; }
    size_t workspace_bytes(int, int, int) override { return 0; }  // the frames are staged in shared memory only
};

int FastBMEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    // bm_fast.cpp:64-65
    if (I0->type != B2F_8UC1 || I1->type != B2F_8UC1) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    const int sw = P.search_window, bw = P.block_window;
    if (sw < 1 || sw > FBM_MAX_SEARCH || bw < 1 || bw > FBM_MAX_BLOCK || (bw & 1) == 0) return B2F_BAD_ARG;
    if (I0->step < (size_t)I0->cols || I1->step < (size_t)I1->cols || !flow_step_ok(flow)) return B2F_BAD_ARG;
    const int rows = I0->rows, cols = I0->cols, br = bw / 2;
    const FbmKeys K = fbm_keys(sw, bw);
    const int ow = 32 - 2 * br;
    const size_t smem = (size_t)(FBM_TH + 2 * br) * 32 + (size_t)(FBM_TH + 2 * br + sw - 1) * (32 + sw - 1);
    const dim3 grid(div_up(cols, ow), div_up(rows, FBM_TH));
    Ctx c = make_ctx(s);
    stats.levels = 1;
    stats.iterations_run = 0;
    const double bytes = 2.0 * rows * cols + 8.0 * rows * cols;
    const bool inter = planar_v == nullptr;
    float *fx = static_cast<float *>(flow->data), *fy = static_cast<float *>(planar_v);
    if (K.wide)
        B2F_LAUNCH(c, 0, bytes, k_fastbm<true>, grid, dim3(FBM_WARPS * 32), smem, static_cast<const uint8_t *>(I0->data),
                   I0->step, static_cast<const uint8_t *>(I1->data), I1->step, rows, cols, fx, flow->step, fy, planar_v_step,
                   inter ? 1 : 0, sw, br, K.bits, K.nq);
    else
        B2F_LAUNCH(c, 0, bytes, k_fastbm<false>, grid, dim3(FBM_WARPS * 32), smem, static_cast<const uint8_t *>(I0->data),
                   I0->step, static_cast<const uint8_t *>(I1->data), I1->step, rows, cols, fx, flow->step, fy, planar_v_step,
                   inter ? 1 : 0, sw, br, K.bits, K.nq);
    active_path_first = 0;
    active_paths.assign(1, (double)(ow | (FBM_TH << 8) | ((K.wide ? 1 : 0) << 16)));
    return finish(c, s);
}

// ------------------------------------------------------------------------------------------- grid BM
constexpr int GBM_WARPS = 8;

// The k-th entry of the reference's spiral scan table (bm.cpp:71-179): rings of radius 1 .. m = min(W, H), each walked
// clockwise from the cell right of its top-left corner; then pairs of whole rows (W < H) or columns (W > H).
__device__ __forceinline__ int2 spiral(int n, int W, int H, int m) {
    int x, y;
    const int rings = 4 * m * (m + 1);
    if (n < rings) {
        int i = (int)((sqrt_approx((float)n + 1.f) - 1.f) * 0.5f);  // an estimate, corrected below
        while (i > 0 && 4 * i * (i + 1) > n) --i;
        while (4 * (i + 1) * (i + 2) <= n) ++i;
        const int r = i + 1, p = n - 4 * i * (i + 1), side = p / (2 * r), t = p - side * 2 * r;
        switch (side) {
            case 0: x = -r + 1 + t; y = -r; break;
            case 1: x = r; y = -r + 1 + t; break;
            case 2: x = r - 1 - t; y = r; break;
            default: x = -r; y = r - 1 - t; break;
        }
        return make_int2(x, y);
    }
    const int q = n - rings;
    if (W < H) {
        const int L = 2 * W + 1, i = m + q / (2 * L), rem = q % (2 * L), side = rem / L;
        x = -m + (rem - side * L);
        y = side ? i + 1 : -(i + 1);
    } else {
        const int L = 2 * H + 1, i = m + q / (2 * L), rem = q % (2 * L), side = rem / L;
        x = side ? i + 1 : -(i + 1);
        y = -m + (rem - side * L);
    }
    return make_int2(x, y);
}

__device__ __forceinline__ int wrap_add(int a, int b) { return (int)((unsigned)a + (unsigned)b); }

__global__ void __launch_bounds__(GBM_WARPS * 32) k_bm_grid(const uint8_t *__restrict__ prev, size_t ps,
                                                           const uint8_t *__restrict__ curr, size_t cs, float *vx, size_t vxs,
                                                           float *vy, size_t vys, int vrows, int vcols, int bw, int bh,
                                                           int shx, int shy, int use_prev, int maxX, int maxY, int accept,
                                                           int escape, int W, int H, int total) {
    const int cell = blockIdx.x * GBM_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (cell >= vrows * vcols) return;  // whole warps leave together
    const int i = cell / vcols, j = cell - i * vcols;
    auto at = [&](float *base, size_t step) { return reinterpret_cast<float *>(reinterpret_cast<char *>(base) + (size_t)i * step) + j; };
    const int X1 = j * shx, Y1 = i * shy;
    const int offX = use_prev ? __float2int_rn(*at(vx, vxs)) : 0;
    const int offY = use_prev ? __float2int_rn(*at(vy, vys)) : 0;
    // SAD of curr at (X1, Y1) against prev at (X2, Y2): the reference's cmpBlocks gets its frames swapped (bm.cu:56,91,112)
    auto sad = [&](int X2, int Y2) {
        int sum = 0;
        for (int y = 0; y < bh; ++y) {
            const uint8_t *c = curr + (size_t)(Y1 + y) * cs + X1, *p = prev + (size_t)(Y2 + y) * ps + X2;
            for (int x = 0; x < bw; ++x) sum += abs((int)__ldg(c + x) - (int)__ldg(p + x));
        }
        return sum;
    };
    auto in_range = [&](int X2, int Y2) { return 0 <= X2 && X2 <= maxX && 0 <= Y2 && Y2 <= maxY; };

    int dist = INT_MAX;
    {
        const int X2 = wrap_add(X1, offX), Y2 = wrap_add(Y1, offY);
        if (in_range(X2, Y2)) {
            int part = 0;
            for (int t = lane; t < bw * bh; t += 32) {
                const int y = t / bw, x = t - y * bw;
                part += abs((int)__ldg(curr + (size_t)(Y1 + y) * cs + X1 + x) - (int)__ldg(prev + (size_t)(Y2 + y) * ps + X2 + x));
            }
            dist = __reduce_add_sync(FULL, part);
        }
    }
    int count = 1, sumx = offX, sumy = offY;
    if (dist > accept) {
        const int m = min(W, H);
        for (int base = 0; base < total; base += 32) {
            const int n = base + lane;
            const int2 o = n < total ? spiral(n, W, H, m) : make_int2(0, 0);
            const int dx = wrap_add(offX, o.x), dy = wrap_add(offY, o.y);
            const int X2 = wrap_add(X1, dx), Y2 = wrap_add(Y1, dy);
            const bool valid = n < total && in_range(X2, Y2);
            const int tmp = valid ? sad(X2, Y2) : INT_MAX;
            const unsigned acc = __ballot_sync(FULL, valid && tmp < accept);
            const int lim = acc ? __ffs(acc) - 1 : 32;  // candidates after the first accepted one are never scanned
            const bool seen = valid && lane < lim;
            if (__ballot_sync(FULL, seen)) {
                const int mn = __reduce_min_sync(FULL, seen ? tmp : INT_MAX);
                if (mn <= dist) {
                    const bool tie = seen && tmp == mn;
                    const int tx = (int)__reduce_add_sync(FULL, tie ? (unsigned)dx : 0u);
                    const int ty = (int)__reduce_add_sync(FULL, tie ? (unsigned)dy : 0u);
                    const int tc = __popc(__ballot_sync(FULL, tie));
                    if (mn < dist) {
                        dist = mn;
                        sumx = tx;
                        sumy = ty;
                        count = tc;
                    } else {
                        sumx = wrap_add(sumx, tx);
                        sumy = wrap_add(sumy, ty);
                        count += tc;
                    }
                }
            }
            if (acc) {
                sumx = __shfl_sync(FULL, dx, lim);
                sumy = __shfl_sync(FULL, dy, lim);
                count = 1;
                break;
            }
        }
        if (dist > escape) {  // dist is the best before any accepted candidate (bm.cu:141-146)
            sumx = offX;
            sumy = offY;
            count = 1;
        }
    }
    if (lane != 0) return;
    const float qx = __fdiv_rn(__int2float_rn(sumx), __int2float_rn(count));
    const float qy = __fdiv_rn(__int2float_rn(sumy), __int2float_rn(count));
    // the division's slow path is a call: the cell index is read again after it rather than kept (and spilled) across it
    unsigned bx, tx;
    asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(bx));
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tx));
    const int c2 = (int)bx * GBM_WARPS + (int)(tx >> 5), i2 = c2 / vcols, j2 = c2 - i2 * vcols;
    reinterpret_cast<float *>(reinterpret_cast<char *>(vx) + (size_t)i2 * vxs)[j2] = qx;
    reinterpret_cast<float *>(reinterpret_cast<char *>(vy) + (size_t)i2 * vys)[j2] = qy;
}

}  // namespace
}  // namespace b2f

extern "C" {

void b2f_fastbm_default_params(b2f_fastbm_params *p) {
    if (!p) return;
    p->search_window = 21;
    p->block_window = 7;
}

int b2f_fastbm_create(const b2f_fastbm_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_fastbm_params d;
    b2f_fastbm_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::FastBMEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

int b2f_calc_optical_flow_bm_size(int rows, int cols, int block_width, int block_height, int shift_width, int shift_height,
                                  int max_range_width, int max_range_height, int *vel_rows, int *vel_cols, int *table_len) {
    if (rows <= 0 || cols <= 0 || block_width < 1 || block_height < 1 || shift_width < 1 || shift_height < 1 ||
        max_range_width < 0 || max_range_height < 0 || max_range_width > B2F_BM_MAX_RANGE ||
        max_range_height > B2F_BM_MAX_RANGE)
        return B2F_BAD_ARG;
    if ((long long)block_width * block_height * 128 > INT_MAX) return B2F_BAD_ARG;  // escapeLevel (bm.cpp:189-197)
    const int vc = (cols - block_width + shift_width) / shift_width;  // bm.cpp:65-66, C division
    const int vr = (rows - block_height + shift_height) / shift_height;
    if (vc <= 0 || vr <= 0) return B2F_BAD_ARG;
    if (vel_rows) *vel_rows = vr;
    if (vel_cols) *vel_cols = vc;
    if (table_len) *table_len = (2 * max_range_width + 1) * (2 * max_range_height + 1) - 1;
    return B2F_OK;
}

int b2f_calc_optical_flow_bm(const b2f_image *prev, const b2f_image *curr, int block_width, int block_height,
                             int shift_width, int shift_height, int max_range_width, int max_range_height, int use_previous,
                             b2f_image *velx, b2f_image *vely, void *cuda_stream) {
    if (!prev || !curr || !velx || !vely || !prev->data || !curr->data || !velx->data || !vely->data) return B2F_BAD_ARG;
    if (prev->rows <= 0 || prev->cols <= 0) return B2F_BAD_ARG;
    if (prev->type != B2F_8UC1 || curr->type != B2F_8UC1) return B2F_UNSUPPORTED_TYPE;  // bm.cpp:62-63
    if (curr->rows != prev->rows || curr->cols != prev->cols) return B2F_SIZE_MISMATCH;
    if (velx->type != B2F_32FC1 || vely->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
    int vr = 0, vc = 0, total = 0;
    int st = b2f_calc_optical_flow_bm_size(prev->rows, prev->cols, block_width, block_height, shift_width, shift_height,
                                           max_range_width, max_range_height, &vr, &vc, &total);
    if (st != B2F_OK) return st;
    if (velx->rows != vr || velx->cols != vc || vely->rows != vr || vely->cols != vc) return B2F_SIZE_MISMATCH;
    if (prev->step < (size_t)prev->cols || curr->step < (size_t)curr->cols || velx->step < (size_t)vc * 4 ||
        vely->step < (size_t)vc * 4)
        return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    b2f::DeviceScope dev(prev->data, s);
    const int area = block_width * block_height;
    const int cells = vr * vc;
    b2f::k_bm_grid<<<b2f::div_up(cells, b2f::GBM_WARPS), b2f::GBM_WARPS * 32, 0, s>>>(
        static_cast<const uint8_t *>(prev->data), prev->step, static_cast<const uint8_t *>(curr->data), curr->step,
        static_cast<float *>(velx->data), velx->step, static_cast<float *>(vely->data), vely->step, vr, vc, block_width,
        block_height, shift_width, shift_height, use_previous ? 1 : 0, prev->cols - block_width, prev->rows - block_height,
        2 * area, 128 * area, max_range_width, max_range_height, total);
    cudaError_t e = cudaPeekAtLastError();
    if (e == cudaSuccess && s == nullptr) e = cudaDeviceSynchronize();  // legacy-stream contract, as b2f_calc
    if (e != cudaSuccess) {
        cudaGetLastError();
        return e == cudaErrorMemoryAllocation ? B2F_OUT_OF_MEMORY : B2F_CUDA_ERROR;
    }
    return B2F_OK;
}

}  // extern "C"
