// dis.cu -- cv::DISOpticalFlow (opencv's video module, dense inverse search) for sm_90a.
//
// oracle/dis_model.py states what these kernels compute; this file is compiled with -fmad=false (csrc/Makefile), so
// every operator rounds once and the float model follows the engine bit for bit.  Spatial propagation is the one of
// OpenCV's OpenCL kernels (a forward scan of every patch row, a descent of every patch, a backward scan, a second
// descent), not the one of its CPU path, which interleaves propagation and descent patch by patch: with propagation on,
// the engine and cv2's CPU class agree statistically, not bit for bit.  The refinement stage is the
// VariationalRefinement solver DeepFlow runs (variational.cuh) with DIS's parameters.
//
// Per pair: the finest level of both frames (1 launch, from the caller's images), then, inside the handle's CUDA graph,
// every coarser level (1 each), and per level Sobel (1) + patch structure tensor (1), the patch search (with
// propagation: scan + descent + scan + descent, else one descent), densification (1), the refinement (as DeepFlow's per
// level) and prolongation (1); last the resize to the frame (1) and the interleave into the caller's flow (1).
//
// Kernel classes: 0 scan (serial along each patch row: latency-bound, one warp per row, two patch SSDs per step),
// 1 descent (one patch per 8 lanes, one lane per patch row, sums reduced by shuffles), 2 densification (per pixel),
// 3 refinement, 4 pyramid / gradients / resize.
#include "variational.cuh"

#include <new>
#include <vector>

namespace b2f {

namespace {

enum { DCLS_SCAN = 0, DCLS_DESCENT = 1, DCLS_DENSE = 2, DCLS_REFINE = 3, DCLS_PYR = 4 };
constexpr int PS = 8, BORDER = 16;
constexpr float DIS_EPS = 0.001f, INV_N = 1.0f / 64.0f;
constexpr unsigned FULL = 0xffffffffu;
// weights per axis: levels have at least PS rows and columns, so a ratio of at most 2^MAX_FINEST (PS + 1) / PS;
// its whole cells plus a partial cell at each end
constexpr int MAX_FINEST = 5, AREA_TAB = (1 << MAX_FINEST) * (PS + 1) / PS + 3;

// ---------------------------------------------------------------------------------------------
// pyramid: cv::resize(INTER_AREA) of u8 frames to about half size (or the caller's frame to 1 / 2^finest).  Exact
// halves: the rounded box mean (a + b + c + d + 2) >> 2.  Otherwise OpenCV's area filter: per axis the weights of
// computeResizeAreaTab (double, stored as float), per source row buf = sum src * alpha, rows summed as b0 buf0 + b1 buf1
// ..., rounded half to even.  Levels are held in float planes of integer values.
// ---------------------------------------------------------------------------------------------
struct U8Src {
    const unsigned char *p;
    size_t step;
    __device__ __forceinline__ float operator()(int y, int x) const { return (float)p[(size_t)y * step + x]; }
};
struct PlaneSrc {
    Plane p;
    __device__ __forceinline__ float operator()(int y, int x) const { return p.at(y, x); }
};

__device__ __forceinline__ int area_tab(int d, int ns, int nd, int *idx, float *wt) {
    const double scale = 1.0 / ((double)nd / ns);
    const double f1 = d * scale, f2 = f1 + scale, cw = fmin(scale, ns - f1);
    int s1 = (int)ceil(f1), s2 = (int)floor(f2);
    s2 = min(s2, ns - 1);
    s1 = min(s1, s2);
    int k = 0;
    if (s1 - f1 > 1e-3) { idx[k] = s1 - 1; wt[k++] = (float)((s1 - f1) / cw); }
    for (int s = s1; s < s2; ++s) { idx[k] = s; wt[k++] = (float)(1.0 / cw); }
    if (f2 - s2 > 1e-3) { idx[k] = s2; wt[k++] = (float)(fmin(fmin(f2 - s2, 1.0), cw) / cw); }
    return k;
}

template <class Src>
__device__ __forceinline__ float area_value(const Src &s, int sh, int sw, int y, int x, int dh, int dw) {
    if (sh == dh && sw == dw) return s(y, x);
    if (sh == 2 * dh && sw == 2 * dw) {
        const int a = (int)s(2 * y, 2 * x), b = (int)s(2 * y, 2 * x + 1), c = (int)s(2 * y + 1, 2 * x),
                  d = (int)s(2 * y + 1, 2 * x + 1);
        return (float)((a + b + c + d + 2) >> 2);
    }
    int xi[AREA_TAB], yi[AREA_TAB];
    float xw[AREA_TAB], yw[AREA_TAB];
    const int nx = area_tab(x, sw, dw, xi, xw), ny = area_tab(y, sh, dh, yi, yw);
    float acc = 0.f;
    for (int b = 0; b < ny; ++b) {
        float buf = 0.f;
        for (int a = 0; a < nx; ++a) buf = buf + s(yi[b], xi[a]) * xw[a];
        acc = b == 0 ? yw[b] * buf : acc + yw[b] * buf;
    }
    return fminf(fmaxf(rintf(acc), 0.f), 255.f);
}

__global__ void __launch_bounds__(256) k_dis_area_u8(U8Src s0, U8Src s1, int sh, int sw, Plane d0, Plane d1, int dh, int dw) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    (blockIdx.z ? d1 : d0).at(y, x) = area_value(blockIdx.z ? s1 : s0, sh, sw, y, x, dh, dw);
}
__global__ void __launch_bounds__(256) k_dis_area(PlaneSrc s0, PlaneSrc s1, int sh, int sw, Plane d0, Plane d1, int dh, int dw) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    (blockIdx.z ? d1 : d0).at(y, x) = area_value(blockIdx.z ? s1 : s0, sh, sw, y, x, dh, dw);
}

// ---------------------------------------------------------------------------------------------
// cv::spatialGradient: 3x3 Sobel of I0, reflect-101 border (integers, exact in float)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int refl101(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return i;
}
__global__ void __launch_bounds__(256) k_dis_sobel(Plane I, Plane gx, Plane gy, int h, int w) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int xl = refl101(x - 1, w), xr = refl101(x + 1, w), yu = refl101(y - 1, h), yd = refl101(y + 1, h);
    const int a = (int)I.at(yu, xl), b = (int)I.at(yu, x), c = (int)I.at(yu, xr);
    const int d = (int)I.at(y, xl), f = (int)I.at(y, xr);
    const int g = (int)I.at(yd, xl), hh = (int)I.at(yd, x), k = (int)I.at(yd, xr);
    gx.at(y, x) = (float)((c + 2 * f + k) - (a + 2 * d + g));
    gy.at(y, x) = (float)((g + 2 * hh + k) - (a + 2 * b + c));
}

// per patch: xx, yy, xy, x, y as exact integer sums over the 8x8 patch, rounded once to float
struct Tensor {
    Plane xx, yy, xy, x, y;
};
__global__ void __launch_bounds__(256) k_dis_tensor(Plane gx, Plane gy, Tensor T, int hs, int ws, int stride) {
    const int js = blockIdx.x * blockDim.x + threadIdx.x, is = blockIdx.y * blockDim.y + threadIdx.y;
    if (js >= ws || is >= hs) return;
    int sxx = 0, syy = 0, sxy = 0, sx = 0, sy = 0;
    for (int r = 0; r < PS; ++r)
        for (int c = 0; c < PS; ++c) {
            const int a = (int)gx.at(is * stride + r, js * stride + c), b = (int)gy.at(is * stride + r, js * stride + c);
            sxx += a * a;
            syy += b * b;
            sxy += a * b;
            sx += a;
            sy += b;
        }
    T.xx.at(is, js) = (float)sxx;
    T.yy.at(is, js) = (float)syy;
    T.xy.at(is, js) = (float)sxy;
    T.x.at(is, js) = (float)sx;
    T.y.at(is, js) = (float)sy;
}

// ---------------------------------------------------------------------------------------------
// One patch at flow (ux, uy), evaluated by 8 lanes (lane r = patch row r).  I1 is sampled from the level extended by
// BORDER replicated pixels (clamped reads), at the clamped position of dis_flow's INIT_BILINEAR_WEIGHTS.  Each lane sums
// its row left to right; xor-shuffles over 4, 2, 1 give every lane ((r0 + r4) + (r2 + r6)) + ((r1 + r5) + (r3 + r7)).
// ---------------------------------------------------------------------------------------------
struct LevelView {
    Plane I0, I1, gx, gy;
    int h, w;
};
__device__ __forceinline__ float row_sum_reduce(float v) {
    v = v + __shfl_xor_sync(FULL, v, 4);
    v = v + __shfl_xor_sync(FULL, v, 2);
    v = v + __shfl_xor_sync(FULL, v, 1);
    return v;
}
template <bool GRADS>
__device__ __forceinline__ void patch_terms(const LevelView &L, int i, int j, float ux, float uy, int r, float &sd,
                                            float &sq, float &sgx, float &sgy) {
    const float yI = fminf(fmaxf(((float)i + uy) + (float)BORDER, (float)(BORDER - PS + 1)), (float)(BORDER + L.h - 1));
    const float xI = fminf(fmaxf(((float)j + ux) + (float)BORDER, (float)(BORDER - PS + 1)), (float)(BORDER + L.w - 1));
    const float di = yI - floorf(yI), dj = xI - floorf(xI);
    const float w11 = di * dj, w10 = di * (1.f - dj), w01 = (1.f - di) * dj, w00 = (1.f - di) * (1.f - dj);
    const int r0 = (int)yI + r, c0 = (int)xI;
    const int ya = clampi(r0 - BORDER, 0, L.h - 1), yb = clampi(r0 + 1 - BORDER, 0, L.h - 1);
    float a = L.I1.at(ya, clampi(c0 - BORDER, 0, L.w - 1)), c = L.I1.at(yb, clampi(c0 - BORDER, 0, L.w - 1));
    float s_d = 0.f, s_q = 0.f, s_x = 0.f, s_y = 0.f;
#pragma unroll
    for (int k = 0; k < PS; ++k) {
        const int xc = clampi(c0 + k + 1 - BORDER, 0, L.w - 1);
        const float b = L.I1.at(ya, xc), d = L.I1.at(yb, xc);
        const float diff = (((w00 * a + w01 * b) + w10 * c) + w11 * d) - L.I0.at(i + r, j + k);
        if (k == 0) {
            s_d = diff;
            s_q = diff * diff;
            if (GRADS) {
                s_x = diff * L.gx.at(i + r, j + k);
                s_y = diff * L.gy.at(i + r, j + k);
            }
        } else {
            s_d = s_d + diff;
            s_q = s_q + diff * diff;
            if (GRADS) {
                s_x = s_x + diff * L.gx.at(i + r, j + k);
                s_y = s_y + diff * L.gy.at(i + r, j + k);
            }
        }
        a = b;
        c = d;
    }
    sd = row_sum_reduce(s_d);
    sq = row_sum_reduce(s_q);
    if (GRADS) {
        sgx = row_sum_reduce(s_x);
        sgy = row_sum_reduce(s_y);
    }
}
__device__ __forceinline__ float patch_ssd(const LevelView &L, int i, int j, float ux, float uy, int r, bool mean_norm) {
    float sd, sq, dummy0, dummy1;
    patch_terms<false>(L, i, j, ux, uy, r, sd, sq, dummy0, dummy1);
    return mean_norm ? sq - (sd * sd) * INV_N : sq;
}

// ---------------------------------------------------------------------------------------------
// Scans: one warp per patch row; lanes 0-7 evaluate one candidate, lanes 8-15 the other (16-31 repeat 0-15), and the
// chain's carried flow stays in registers.  Forward: the patch's own start flow (k_dis_start) against the
// carried one, keep the carried one when its SSD is lower.  Backward: the patch's flow against its right neighbour's
// (already chosen), take the neighbour's when its SSD is lower.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_dis_scan_fwd(LevelView L, Plane Sx, Plane Sy, int hs, int ws, int stride,
                                                      int mean_norm) {
    const int is = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31, r = lane & 7, cand = (lane >> 3) & 1;
    if (is >= hs) return;  // whole warps
    const int i = is * stride;
    float px = Sx.at(is, 0), py = Sy.at(is, 0);
    for (int js = 1; js < ws; ++js) {
        const int j = js * stride;
        const float ox = Sx.at(is, js), oy = Sy.at(is, js);
        const float e = patch_ssd(L, i, j, cand ? px : ox, cand ? py : oy, r, mean_norm);
        const float e_own = __shfl_sync(FULL, e, 0), e_car = __shfl_sync(FULL, e, 8);
        if (!(e_car < e_own)) {
            px = ox;
            py = oy;
        }
        __syncwarp();  // every lane has read S(is, js) before lane 0 overwrites it
        if (lane == 0) {
            Sx.at(is, js) = px;
            Sy.at(is, js) = py;
        }
    }
}
__global__ void __launch_bounds__(128) k_dis_scan_bwd(LevelView L, Plane Sx, Plane Sy, int hs, int ws, int stride,
                                                      int mean_norm) {
    const int is = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31, r = lane & 7, cand = (lane >> 3) & 1;
    if (is >= hs) return;
    const int i = is * stride;
    float rx = Sx.at(is, ws - 1), ry = Sy.at(is, ws - 1);
    for (int js = ws - 2; js >= 0; --js) {
        const int j = js * stride;
        const float ox = Sx.at(is, js), oy = Sy.at(is, js);
        const float e = patch_ssd(L, i, j, cand ? rx : ox, cand ? ry : oy, r, mean_norm);
        const float e_own = __shfl_sync(FULL, e, 0), e_right = __shfl_sync(FULL, e, 8);
        if (!(e_right < e_own)) {
            rx = ox;
            ry = oy;
        }
        __syncwarp();  // every lane has read S(is, js) before lane 0 overwrites it
        if (lane == 0) {
            Sx.at(is, js) = rx;
            Sy.at(is, js) = ry;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Descent: 8 lanes per patch, 32 patches per CTA.  Inverse compositional steps by the inverse structure tensor; a
// patch stops after the step that did not lower its SSD (the warp keeps evaluating while any of its patches runs, so
// the shuffles always see the full warp); a result farther than the patch size from the start is dropped.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_dis_descent(LevelView L, Tensor T, Plane Sx, Plane Sy, int hs, int ws, int stride,
                                                     int iters, int mean_norm) {
    const int p = blockIdx.x * 32 + (threadIdx.x >> 3), r = threadIdx.x & 7, n = hs * ws;
    const bool valid = p < n;
    const int pc = valid ? p : n - 1;
    const int is = pc / ws, js = pc - is * ws, i = is * stride, j = js * stride;
    const float u0x = Sx.at(is, js), u0y = Sy.at(is, js);
    const float xx = T.xx.at(is, js), yy = T.yy.at(is, js), xy = T.xy.at(is, js);
    const float xs = T.x.at(is, js), ys = T.y.at(is, js);
    const float det = xx * yy - xy * xy;
    const float inv = fabsf(det) < DIS_EPS ? 1.0f / DIS_EPS : 1.0f / det;
    const float h11 = yy * inv, h12 = (-xy) * inv, h22 = xx * inv;
    float cx = u0x, cy = u0y, prev = 1e10f;
    bool active = valid;
    for (int t = 0; t < iters; ++t) {
        if (!__any_sync(FULL, active)) break;
        float sd, sq, gx, gy;
        patch_terms<true>(L, i, j, cx, cy, r, sd, sq, gx, gy);
        if (active) {
            float ssd = sq, dux = gx, duy = gy;
            if (mean_norm) {
                ssd = sq - (sd * sd) * INV_N;
                dux = gx - (sd * xs) * INV_N;
                duy = gy - (sd * ys) * INV_N;
            }
            cx = cx - (h11 * dux + h12 * duy);
            cy = cy - (h12 * dux + h22 * duy);
            if (!(ssd < prev)) active = false;
            prev = ssd;
        }
    }
    if (valid && r == 0) {
        const float vx = cx - u0x, vy = cy - u0y;
        const bool ok = (vx * vx + vy * vy) <= (float)(PS * PS);
        Sx.at(is, js) = ok ? cx : u0x;
        Sy.at(is, js) = ok ? cy : u0y;
    }
}

// Each patch's start: the dense flow at its centre.  With `zero_candidate` (the level that receives the caller's
// initial flow) zero flow replaces it where zero's SSD is lower.  8 lanes per patch, as the descent.
__global__ void __launch_bounds__(256) k_dis_start(LevelView L, Plane Ux, Plane Uy, Plane Sx, Plane Sy, int hs, int ws,
                                                   int stride, int zero_candidate, int mean_norm) {
    const int p = blockIdx.x * 32 + (threadIdx.x >> 3), r = threadIdx.x & 7, n = hs * ws;
    const bool valid = p < n;
    const int pc = valid ? p : n - 1;
    const int is = pc / ws, js = pc - is * ws, i = is * stride, j = js * stride;
    float ux = Ux.at(i + PS / 2, j + PS / 2), uy = Uy.at(i + PS / 2, j + PS / 2);
    if (zero_candidate) {  // uniform over the launch: every lane takes part in the shuffles
        const float e_own = patch_ssd(L, i, j, ux, uy, r, mean_norm), e_zero = patch_ssd(L, i, j, 0.f, 0.f, r, mean_norm);
        if (e_zero < e_own) {
            ux = 0.f;
            uy = 0.f;
        }
    }
    if (valid && r == 0) {
        Sx.at(is, js) = ux;
        Sy.at(is, js) = uy;
    }
}

// ---------------------------------------------------------------------------------------------
// Densification: each pixel averages the flows of the patches that cover it, weighted by 1 / max(1, |I1(x + S) - I0|)
// (I1 bilinear at the clamped moved position), is outer, js inner.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_dis_densify(Plane I0, Plane I1, Plane Sx, Plane Sy, Plane Ux, Plane Uy, int h, int w,
                                                     int stride) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int end_is = min(y / stride, (h - PS) / stride), end_js = min(x / stride, (w - PS) / stride);
    const int start_is = min(max(0, y - PS + stride) / stride, end_is);
    const int start_js = min(max(0, x - PS + stride) / stride, end_js);
    const float lim_x = ((float)w - 1.f) - DIS_EPS, lim_y = ((float)h - 1.f) - DIS_EPS;
    const float i0 = I0.at(y, x);
    float su = 0.f, sv = 0.f, sc = 0.f;
    for (int is = start_is; is <= end_is; ++is)
        for (int js = start_js; js <= end_js; ++js) {
            const float sx = Sx.at(is, js), sy = Sy.at(is, js);
            const float jm = fminf(fmaxf((float)x + sx, 0.f), lim_x), im = fminf(fmaxf((float)y + sy, 0.f), lim_y);
            const int jl = (int)jm, il = (int)im, ju = jl + 1, iu = il + 1;
            const float fjl = (float)jl, fil = (float)il, fju = (float)ju, fiu = (float)iu;
            const float diff = ((((jm - fjl) * (im - fil)) * I1.at(iu, ju) + ((fju - jm) * (im - fil)) * I1.at(iu, jl)) +
                                ((jm - fjl) * (fiu - im)) * I1.at(il, ju)) +
                               ((fju - jm) * (fiu - im)) * I1.at(il, jl) - i0;
            const float coef = 1.f / fmaxf(1.f, fabsf(diff));
            su = su + coef * sx;
            sv = sv + coef * sy;
            sc = sc + coef;
        }
    Ux.at(y, x) = su / sc;
    Uy.at(y, x) = sv / sc;
}

// ---------------------------------------------------------------------------------------------
// host engine
// ---------------------------------------------------------------------------------------------
static int auto_coarsest(int rows, int cols, int ps) {
    const int mn = std::min(rows, cols), mx = std::max(rows, cols);
    if (mn < ps) return -1;
    return std::min(static_cast<int>(std::log(mx / (4.0 * ps)) / std::log(2.0) + 0.5),
                    static_cast<int>(std::log(static_cast<double>(mn / ps)) / std::log(2.0)));
}

static bool same_params(const b2f_dis_params &a, const b2f_dis_params &b) {
    return a.finest_scale == b.finest_scale && a.coarsest_scale == b.coarsest_scale && a.patch_size == b.patch_size &&
           a.patch_stride == b.patch_stride && a.grad_descent_iterations == b.grad_descent_iterations &&
           a.variational_refinement_iterations == b.variational_refinement_iterations && a.alpha == b.alpha &&
           a.delta == b.delta && a.gamma == b.gamma && a.epsilon == b.epsilon &&
           a.use_mean_normalization == b.use_mean_normalization && a.use_spatial_propagation == b.use_spatial_propagation &&
           a.use_initial_flow == b.use_initial_flow;
}

constexpr int REFINE_SOR_ITERATIONS = 5;
constexpr float REFINE_OMEGA = 1.6f;

class DISEngine : public b2f_handle {
public:
    explicit DISEngine(const b2f_dis_params &p) : P(p) { algo = ALGO_DIS; }
    b2f_dis_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    // what cv2.DISOpticalFlow reports: the class does not override getDefaultName
    const char *default_name() const override { return "my_object"; }
    bool reads_flow() const override { return P.use_initial_flow != 0; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"dis_scan", "dis_descent", "dis_densification", "dis_refinement", "dis_pyramid"};
        return (cls >= 0 && cls < 5) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        if (level_sizes(rows, cols).empty()) return 0;
        Layout L;
        return layout(rows, cols, true, L);
    }

private:
    enum { S_GX = 0, S_GY, S_U, S_V, S_UN, S_VN, S_IX, S_IY, S_IZ, S_IXX, S_IXY, S_IYY, S_IXZ, S_IYZ, S_DU, S_DV, S_DUN,
           S_DVN, S_A12, S_B1, S_B2, S_DENU, S_DENV, S_WR, S_WD, S_XX, S_YY, S_XY, S_X, S_Y, S_SX, S_SY, S_COUNT,
           S_AVG = S_A12 };
    struct DLevel {
        int rows = 0, cols = 0;
        Plane I0, I1;
    };
    struct Layout {
        int rows = 0, cols = 0;
        b2f_dis_params P{};
        std::vector<DLevel> levels;  // finest .. coarsest
        float *shared[S_COUNT] = {};
        Plane out_u{}, out_v{};
    };
    Layout L_;
    struct GraphKey {  // the schedule reads no knob
        int rows, cols;
        b2f_dis_params P;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;

    std::vector<std::pair<int, int>> level_sizes(int rows, int cols) const;
    size_t layout(int rows, int cols, bool counting, Layout &L);
    cudaError_t ensure_workspace(int rows, int cols);
    Plane sp(int idx, int cols) const { return Plane{L_.shared[idx], plane_pitch(cols)}; }
    void solve(Ctx &c);
};

// levels finest .. coarsest; empty when the frame cannot hold the finest scale
std::vector<std::pair<int, int>> DISEngine::level_sizes(int rows, int cols) const {
    std::vector<std::pair<int, int>> s;
    int c = auto_coarsest(rows, cols, P.patch_size);
    if (P.coarsest_scale >= 0) c = std::min(c, P.coarsest_scale);
    if (P.finest_scale < 0 || P.finest_scale > MAX_FINEST || c < P.finest_scale) return s;
    s.push_back({rows >> P.finest_scale, cols >> P.finest_scale});
    for (int i = P.finest_scale; i < c; ++i) s.push_back({s.back().first / 2, s.back().second / 2});
    for (const auto &l : s)
        if (l.first < PS || l.second < PS) return {};
    return s;
}

size_t DISEngine::layout(int rows, int cols, bool counting, Layout &L) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.rows = rows;
    L.cols = cols;
    L.P = P;
    L.levels.clear();
    for (const auto &s : level_sizes(rows, cols)) {
        DLevel lv;
        lv.rows = s.first;
        lv.cols = s.second;
        lv.I0 = A.plane(lv.rows, lv.cols);
        lv.I1 = A.plane(lv.rows, lv.cols);
        L.levels.push_back(lv);
    }
    const int fr = L.levels[0].rows, fc = L.levels[0].cols;
    for (int i = 0; i < S_COUNT; ++i) L.shared[i] = A.plane(fr, fc).p;
    L.out_u = A.plane(rows, cols);
    L.out_v = A.plane(rows, cols);
    return A.used();
}

cudaError_t DISEngine::ensure_workspace(int rows, int cols) {
    if (L_.rows == rows && L_.cols == cols && same_params(L_.P, P) && arena.capacity() > 0) return cudaSuccess;
    Layout tmp;
    const size_t need = layout(rows, cols, true, tmp);
    graph_.destroy();
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    layout(rows, cols, false, L_);
    return cudaSuccess;
}

void DISEngine::solve(Ctx &c) {
    const dim3 block(32, 8);
    const int nl = static_cast<int>(L_.levels.size());
    const int st = P.patch_stride, mn = P.use_mean_normalization ? 1 : 0;
    // level 0 (the finest) is written by calc() before this schedule: it reads the caller's images
    for (int l = 1; l < nl; ++l) {
        const DLevel &a = L_.levels[l - 1], &b = L_.levels[l];
        B2F_LAUNCH(c, DCLS_PYR, 2.0 * 4.0 * ((double)a.rows * a.cols + (double)b.rows * b.cols), k_dis_area,
                   dim3(div_up(b.cols, 32), div_up(b.rows, 8), 2), block, 0, PlaneSrc{a.I0}, PlaneSrc{a.I1}, a.rows,
                   a.cols, b.I0, b.I1, b.rows, b.cols);
    }
    DFParams k;
    k.alpha2 = static_cast<float>(P.alpha) * 0.5f;
    k.delta2 = static_cast<float>(P.delta) * 0.5f;
    k.gamma2 = static_cast<float>(P.gamma) * 0.5f;
    k.z2 = ZETA * ZETA;
    k.e2 = static_cast<float>(P.epsilon) * static_cast<float>(P.epsilon);
    k.omega = REFINE_OMEGA;
    k.omo = 1.0f - k.omega;

    int ui = 0;
    {
        const DLevel &lc = L_.levels[nl - 1];
        if (P.use_initial_flow) {
            // the caller's flow (split into out_u / out_v by calc()) resized to the coarsest level, times 1 / 2^scale
            const int scale = P.finest_scale + nl - 1;
            B2F_LAUNCH(c, DCLS_PYR, 2.0 * 4.0 * ((double)L_.rows * L_.cols + (double)lc.rows * lc.cols), k_df_resize,
                       dim3(div_up(lc.cols, 32), div_up(lc.rows, 8), 2), block, 0, L_.out_u, L_.out_v, L_.rows, L_.cols,
                       sp(S_U, lc.cols), sp(S_V, lc.cols), lc.rows, lc.cols, (double)L_.cols / lc.cols,
                       (double)L_.rows / lc.rows, 1.0f / static_cast<float>(1 << scale), 1);
        } else {
            fill_plane(c, sp(S_U, lc.cols), lc.rows, lc.cols, 0.f);
            fill_plane(c, sp(S_V, lc.cols), lc.rows, lc.cols, 0.f);
        }
    }
    for (int l = nl - 1; l >= 0; --l) {
        const DLevel &lv = L_.levels[l];
        const int h = lv.rows, w = lv.cols, hs = 1 + (h - PS) / st, ws = 1 + (w - PS) / st;
        const double npx = (double)h * w, npatch = (double)hs * ws;
        const dim3 grid(div_up(w, 32), div_up(h, 8)), pgrid(div_up(ws, 32), div_up(hs, 8));
        Plane U = sp(ui ? S_UN : S_U, w), V = sp(ui ? S_VN : S_V, w);
        Plane GX = sp(S_GX, w), GY = sp(S_GY, w);
        // the patch planes are (hs, ws); their pitch follows the level's
        Plane SX = sp(S_SX, w), SY = sp(S_SY, w);
        Tensor T{sp(S_XX, w), sp(S_YY, w), sp(S_XY, w), sp(S_X, w), sp(S_Y, w)};
        LevelView LV{lv.I0, lv.I1, GX, GY, h, w};

        B2F_LAUNCH(c, DCLS_PYR, 12.0 * npx, k_dis_sobel, grid, block, 0, lv.I0, GX, GY, h, w);
        B2F_LAUNCH(c, DCLS_PYR, 8.0 * npx + 20.0 * npatch, k_dis_tensor, pgrid, block, 0, GX, GY, T, hs, ws, st);
        // per SSD: 64 I0 + 81 I1 floats (+ 128 gradient floats in the descent), at most the level's pixels from DRAM
        const double scan_bytes = 2.0 * npatch * 145.0 * 4.0, desc_bytes = npatch * (273.0 * 4.0 + 36.0);
        const int desc_blocks = div_up(hs * ws, 32), scan_blocks = div_up(hs, 4);
        const int zero_candidate = P.use_initial_flow && l == nl - 1;
        B2F_LAUNCH(c, DCLS_SCAN, zero_candidate ? scan_bytes : 16.0 * npatch, k_dis_start, dim3(desc_blocks), dim3(256),
                   0, LV, U, V, SX, SY, hs, ws, st, zero_candidate, mn);
        if (P.use_spatial_propagation) {
            B2F_LAUNCH(c, DCLS_SCAN, scan_bytes, k_dis_scan_fwd, dim3(scan_blocks), dim3(128), 0, LV, SX, SY, hs, ws,
                       st, mn);
            B2F_LAUNCH(c, DCLS_DESCENT, desc_bytes, k_dis_descent, dim3(desc_blocks), dim3(256), 0, LV, T, SX, SY, hs,
                       ws, st, P.grad_descent_iterations, mn);
            B2F_LAUNCH(c, DCLS_SCAN, scan_bytes, k_dis_scan_bwd, dim3(scan_blocks), dim3(128), 0, LV, SX, SY, hs, ws,
                       st, mn);
        }
        B2F_LAUNCH(c, DCLS_DESCENT, desc_bytes, k_dis_descent, dim3(desc_blocks), dim3(256), 0, LV, T, SX, SY, hs, ws,
                   st, P.grad_descent_iterations, mn);
        B2F_LAUNCH(c, DCLS_DENSE, 24.0 * npx, k_dis_densify, grid, block, 0, lv.I0, lv.I1, SX, SY, U, V, h, w, st);

        int it = 0;
        if (P.variational_refinement_iterations > 0) {
            LevelPlanes R;
            R.Ix = sp(S_IX, w); R.Iy = sp(S_IY, w); R.Iz = sp(S_IZ, w);
            R.Ixx = sp(S_IXX, w); R.Ixy = sp(S_IXY, w); R.Iyy = sp(S_IYY, w); R.Ixz = sp(S_IXZ, w); R.Iyz = sp(S_IYZ, w);
            R.u = U; R.v = V;
            R.du = sp(S_DU, w); R.dv = sp(S_DV, w);
            R.a12 = sp(S_A12, w); R.b1 = sp(S_B1, w); R.b2 = sp(S_B2, w);
            R.den_u = sp(S_DENU, w); R.den_v = sp(S_DENV, w); R.wr = sp(S_WR, w); R.wd = sp(S_WD, w);
            it = variational_iters_per_launch(REFINE_SOR_ITERATIONS, h, w, sm_count());
            variational_level(c, R, lv.I0, lv.I1, sp(S_AVG, w), sp(S_DUN, w), sp(S_DVN, w), h, w, k,
                              P.variational_refinement_iterations, REFINE_SOR_ITERATIONS, it, DCLS_REFINE, DCLS_REFINE,
                              DCLS_REFINE, DCLS_REFINE);
        }
        // bits 0-7: refinement SOR iterations per solver launch; bits 8-23: hs; 24-39: ws
        active_paths[l] = (double)it + 256.0 * ((double)hs + 65536.0 * (double)ws);
        if (l > 0) {
            const DLevel &nx = L_.levels[l - 1];
            Plane nu = sp(ui ? S_U : S_UN, nx.cols), nv = sp(ui ? S_V : S_VN, nx.cols);
            B2F_LAUNCH(c, DCLS_PYR, 2.0 * 4.0 * (npx + (double)nx.rows * nx.cols), k_df_resize,
                       dim3(div_up(nx.cols, 32), div_up(nx.rows, 8), 2), block, 0, U, V, h, w, nu, nv, nx.rows,
                       nx.cols, (double)w / nx.cols, (double)h / nx.rows, 2.0f, 1);
            ui ^= 1;
        }
    }
    const DLevel &f = L_.levels[0];
    B2F_LAUNCH(c, DCLS_PYR, 2.0 * 4.0 * ((double)f.rows * f.cols + (double)L_.rows * L_.cols), k_df_resize,
               dim3(div_up(L_.cols, 32), div_up(L_.rows, 8), 2), block, 0, sp(ui ? S_UN : S_U, f.cols),
               sp(ui ? S_VN : S_V, f.cols), f.rows, f.cols, L_.out_u, L_.out_v, L_.rows, L_.cols,
               (double)f.cols / L_.cols, (double)f.rows / L_.rows, static_cast<float>(1 << P.finest_scale), 1);
}

int DISEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    if (I0->type != B2F_8UC1 || I1->type != B2F_8UC1) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    // patch size 8 is the only one built (all three presets use it)
    if (P.patch_size != PS || P.patch_stride < 1 || P.patch_stride > P.patch_size || P.grad_descent_iterations < 0 ||
        P.variational_refinement_iterations < 0 || !(P.alpha >= 0.0) || !(P.delta >= 0.0) || !(P.gamma >= 0.0) ||
        !(P.epsilon > 0.0))
        return B2F_BAD_ARG;
    if (I0->step < (size_t)I0->cols || I1->step < (size_t)I1->cols || !flow_step_ok(flow)) return B2F_BAD_ARG;
    const int rows = I0->rows, cols = I0->cols;
    if (level_sizes(rows, cols).empty()) return B2F_BAD_ARG;
    Ctx c = make_ctx(s);
    static DeviceOnce attrs;
    attrs.run(c, [&] {
        c.check(cudaFuncSetAttribute(k_df_sor, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(sizeof(float) * SOR_PLANES * SR * SR)));
    });
    c.check(ensure_workspace(rows, cols));
    if (!c.ok()) return finish(c, s);
    stats.levels = static_cast<int>(L_.levels.size());
    stats.iterations_run = 0;
    active_paths.assign(L_.levels.size(), 0.0);  // level l is pyramid scale finest_scale + l
    active_path_first = P.finest_scale;

    const ImageView vf = flow_view(flow, rows, cols);
    if (P.use_initial_flow) split_flow(c, DCLS_PYR, vf, L_.out_u, L_.out_v);  // read before the graph: the caller's buffer
    {
        const DLevel &f = L_.levels[0];
        B2F_LAUNCH(c, DCLS_PYR, 2.0 * ((double)rows * cols + 4.0 * f.rows * f.cols), k_dis_area_u8,
                   dim3(div_up(f.cols, 32), div_up(f.rows, 8), 2), dim3(32, 8), 0,
                   U8Src{static_cast<const unsigned char *>(I0->data), I0->step},
                   U8Src{static_cast<const unsigned char *>(I1->data), I1->step}, rows, cols, f.I0, f.I1, f.rows, f.cols);
    }
    const bool want_graph = knobs.use_graph && !profiling && s != nullptr;
    if (want_graph) {
        graph_.run(*this, c, s, GraphKey{rows, cols, P, L_.levels[0].I0.p}, [&](Ctx &g) { solve(g); });
    } else {
        solve(c);
    }
    merge_flow(c, DCLS_PYR, L_.out_u, L_.out_v, vf);
    return finish(c, s);
}

int DISEngine::set_param(int id, double v) {
    switch (id) {
        case B2F_DIS_FINEST_SCALE: P.finest_scale = static_cast<int>(v); break;
        case B2F_DIS_COARSEST_SCALE: P.coarsest_scale = static_cast<int>(v); break;
        case B2F_DIS_PATCH_SIZE: P.patch_size = static_cast<int>(v); break;
        case B2F_DIS_PATCH_STRIDE: P.patch_stride = static_cast<int>(v); break;
        case B2F_DIS_GRADIENT_DESCENT_ITERATIONS: P.grad_descent_iterations = static_cast<int>(v); break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_ITERATIONS: P.variational_refinement_iterations = static_cast<int>(v); break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_ALPHA: P.alpha = v; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_DELTA: P.delta = v; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_GAMMA: P.gamma = v; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_EPSILON: P.epsilon = v; break;
        case B2F_DIS_USE_MEAN_NORMALIZATION: P.use_mean_normalization = v != 0.0; break;
        case B2F_DIS_USE_SPATIAL_PROPAGATION: P.use_spatial_propagation = v != 0.0; break;
        case B2F_DIS_USE_INITIAL_FLOW: P.use_initial_flow = v != 0.0; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

int DISEngine::get_param(int id, double *v) const {
    switch (id) {
        case B2F_DIS_FINEST_SCALE: *v = P.finest_scale; break;
        case B2F_DIS_COARSEST_SCALE: *v = P.coarsest_scale; break;
        case B2F_DIS_PATCH_SIZE: *v = P.patch_size; break;
        case B2F_DIS_PATCH_STRIDE: *v = P.patch_stride; break;
        case B2F_DIS_GRADIENT_DESCENT_ITERATIONS: *v = P.grad_descent_iterations; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_ITERATIONS: *v = P.variational_refinement_iterations; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_ALPHA: *v = P.alpha; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_DELTA: *v = P.delta; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_GAMMA: *v = P.gamma; break;
        case B2F_DIS_VARIATIONAL_REFINEMENT_EPSILON: *v = P.epsilon; break;
        case B2F_DIS_USE_MEAN_NORMALIZATION: *v = P.use_mean_normalization; break;
        case B2F_DIS_USE_SPATIAL_PROPAGATION: *v = P.use_spatial_propagation; break;
        case B2F_DIS_USE_INITIAL_FLOW: *v = P.use_initial_flow; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

}  // namespace

}  // namespace b2f

extern "C" {

void b2f_dis_default_params(b2f_dis_params *p, int preset) {
    if (!p) return;
    p->finest_scale = 2;
    p->coarsest_scale = -1;
    p->patch_size = 8;
    p->patch_stride = 4;
    p->grad_descent_iterations = 16;
    p->variational_refinement_iterations = 5;
    p->alpha = 20.0;
    p->delta = 5.0;
    p->gamma = 10.0;
    p->epsilon = 0.01;
    p->use_mean_normalization = 1;
    p->use_spatial_propagation = 1;
    p->use_initial_flow = 0;
    if (preset == B2F_DIS_PRESET_ULTRAFAST) {
        p->grad_descent_iterations = 12;
        p->variational_refinement_iterations = 0;
    } else if (preset == B2F_DIS_PRESET_MEDIUM) {
        p->finest_scale = 1;
        p->patch_stride = 3;
        p->grad_descent_iterations = 25;
    }
}

int b2f_dis_create(const b2f_dis_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_dis_params d;
    b2f_dis_default_params(&d, B2F_DIS_PRESET_FAST);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::DISEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
