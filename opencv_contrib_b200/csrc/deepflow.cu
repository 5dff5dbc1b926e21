// deepflow.cu -- cv::optflow::createOptFlow_DeepFlow (modules/optflow/src/deepflow.cpp) for sm_90a.
//
// deepflow.cpp is a driver: 3x3 Gaussian pre-smoothing, a pyramid with a 0.95 step built by cv::resize, and one
// cv::VariationalRefinement call per level, coarse to fine.  The reference has no GPU implementation.  The
// discretization of VariationalRefinement is the one oracle/deepflow_model.py states (established by probing cv2 and
// pinned against it per call); these kernels evaluate the same float32 expressions in the same order.  The solver's
// kernels live in variational.cuh, which the DIS engine (dis.cu) shares.  This file is
// compiled with -fmad=false (csrc/Makefile), so every operator below rounds once and the float model follows the
// engine bit for bit; division and square root are the IEEE ones (no fast-math).
//
// Per pair: pre-smoothing (1 launch), pyramid (one resize per level), then per level: warp (1) + derivatives (1), per
// fixed-point step one system-terms launch and ceil(sor / k) solver launches, and one add + prolongation.  A level that
// fits one 64x64 region runs all its fixed-point steps in one single-CTA launch.
//
// Kernel classes: 0 sor (44 B/px algorithmic per SOR iteration), 1 system terms (88 B/px), 2 warp + derivatives,
// 3 pyramid (conversion, smoothing, resize, add).
#include "variational.cuh"

#include <new>
#include <vector>

namespace b2f {

namespace {

// ---------------------------------------------------------------------------------------------
// host engine
// ---------------------------------------------------------------------------------------------
struct DLevel {
    int rows = 0, cols = 0;
    Plane I0, I1;
};

// deepflow.cpp buildPyramid: next = (int)(prev * 0.95f + 0.5f) in float, stop when a side is <= minSize; the source plus
// at most maxLayers levels below it
static std::vector<std::pair<int, int>> pyramid_sizes(int rows, int cols, const b2f_deepflow_params &p) {
    std::vector<std::pair<int, int>> s{{rows, cols}};
    const float f = static_cast<float>(p.downscale_factor);
    for (int i = 0; i < p.max_layers; ++i) {
        const int nc = static_cast<int>(static_cast<float>(s.back().second) * f + 0.5f);
        const int nr = static_cast<int>(static_cast<float>(s.back().first) * f + 0.5f);
        if (nr <= p.min_size || nc <= p.min_size) break;
        s.push_back({nr, nc});
    }
    return s;
}

static bool same_params(const b2f_deepflow_params &a, const b2f_deepflow_params &b) {
    return a.sigma == b.sigma && a.min_size == b.min_size && a.downscale_factor == b.downscale_factor &&
           a.fixed_point_iterations == b.fixed_point_iterations && a.sor_iterations == b.sor_iterations &&
           a.alpha == b.alpha && a.delta == b.delta && a.gamma == b.gamma && a.omega == b.omega &&
           a.max_layers == b.max_layers;
}

class DeepFlowEngine : public b2f_handle {
public:
    explicit DeepFlowEngine(const b2f_deepflow_params &p) : P(p) { algo = ALGO_DEEPFLOW; }
    b2f_deepflow_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    // the reference class does not override getDefaultName; this is the name the engine reports
    const char *default_name() const override { return "DenseOpticalFlow.DeepFlow"; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"deepflow_sor", "deepflow_terms", "deepflow_warp_derivatives", "deepflow_pyramid"};
        return (cls >= 0 && cls < 4) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        Layout L;
        return layout(rows, cols, true, L);
    }

private:
    // the average of I0 and the warped I1 (S_AVG) is dead once the derivatives are written: it shares A12's plane
    enum { S_IX = 0, S_IY, S_IZ, S_IXX, S_IXY, S_IYY, S_IXZ, S_IYZ, S_U, S_V, S_UN, S_VN, S_DU, S_DV,
           S_DUN, S_DVN, S_A12, S_B1, S_B2, S_DENU, S_DENV, S_WR, S_WD, S_COUNT, S_AVG = S_A12 };
    struct Layout {
        int rows = 0, cols = 0;
        b2f_deepflow_params P{};
        std::vector<DLevel> levels;
        float *shared[S_COUNT] = {};
    };
    Layout L_;
    struct GraphKey {  // the schedule reads no knob
        int rows, cols;
        b2f_deepflow_params P;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;
    int final_ui_ = 0;

    size_t layout(int rows, int cols, bool counting, Layout &L);
    cudaError_t ensure_workspace(int rows, int cols);
    Plane sp(int idx, int cols) const { return Plane{L_.shared[idx], plane_pitch(cols)}; }
    void solve(Ctx &c);
};

size_t DeepFlowEngine::layout(int rows, int cols, bool counting, Layout &L) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.rows = rows;
    L.cols = cols;
    L.P = P;
    L.levels.clear();
    for (const auto &s : pyramid_sizes(rows, cols, P)) {
        DLevel lv;
        lv.rows = s.first;
        lv.cols = s.second;
        lv.I0 = A.plane(lv.rows, lv.cols);
        lv.I1 = A.plane(lv.rows, lv.cols);
        L.levels.push_back(lv);
    }
    for (int i = 0; i < S_COUNT; ++i) L.shared[i] = A.plane(rows, cols).p;
    return A.used();
}

cudaError_t DeepFlowEngine::ensure_workspace(int rows, int cols) {
    if (L_.rows == rows && L_.cols == cols && same_params(L_.P, P) && arena.capacity() > 0) return cudaSuccess;
    Layout tmp;
    const size_t need = layout(rows, cols, true, tmp);
    graph_.destroy();
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    layout(rows, cols, false, L_);
    return cudaSuccess;
}

void DeepFlowEngine::solve(Ctx &c) {
    const dim3 block(32, 8);
    const int nl = static_cast<int>(L_.levels.size());
    // level 0 (the smoothed frames) is written by calc() before this schedule: it reads the caller's images, which a
    // captured graph must not bake in
    for (int l = 1; l < nl; ++l) {
        const DLevel &a = L_.levels[l - 1], &b = L_.levels[l];
        B2F_LAUNCH(c, CLS_PYR, 2.0 * 4.0 * ((double)a.rows * a.cols + (double)b.rows * b.cols), k_df_resize,
                   dim3(div_up(b.cols, 32), div_up(b.rows, 8), 2), block, 0, a.I0, a.I1, a.rows, a.cols, b.I0, b.I1, b.rows,
                   b.cols, (double)a.cols / b.cols, (double)a.rows / b.rows, 1.0f, 0);
    }
    DFParams k;
    k.alpha2 = static_cast<float>(4.0f * static_cast<float>(P.alpha)) * 0.5f;
    k.delta2 = (static_cast<float>(P.delta) / 3.0f) * 0.5f;
    k.gamma2 = (static_cast<float>(P.gamma) / 3.0f) * 0.5f;
    k.z2 = ZETA * ZETA;
    k.e2 = EPSILON * EPSILON;
    k.omega = static_cast<float>(P.omega);
    k.omo = 1.0f - k.omega;
    const float mul = 1.0f / static_cast<float>(P.downscale_factor);

    int ui = 0;
    {
        const DLevel &lc = L_.levels[nl - 1];
        fill_plane(c, sp(S_U, lc.cols), lc.rows, lc.cols, 0.f);
        fill_plane(c, sp(S_V, lc.cols), lc.rows, lc.cols, 0.f);
    }
    for (int l = nl - 1; l >= 0; --l) {
        const DLevel &lv = L_.levels[l];
        const int h = lv.rows, w = lv.cols;
        const double npx = (double)h * w;
        LevelPlanes T;
        T.Ix = sp(S_IX, w); T.Iy = sp(S_IY, w); T.Iz = sp(S_IZ, w);
        T.Ixx = sp(S_IXX, w); T.Ixy = sp(S_IXY, w); T.Iyy = sp(S_IYY, w); T.Ixz = sp(S_IXZ, w); T.Iyz = sp(S_IYZ, w);
        T.u = sp(ui ? S_UN : S_U, w); T.v = sp(ui ? S_VN : S_V, w);
        T.du = sp(S_DU, w); T.dv = sp(S_DV, w);
        T.a12 = sp(S_A12, w); T.b1 = sp(S_B1, w); T.b2 = sp(S_B2, w);
        T.den_u = sp(S_DENU, w); T.den_v = sp(S_DENV, w); T.wr = sp(S_WR, w); T.wd = sp(S_WD, w);
        const int it = variational_iters_per_launch(P.sor_iterations, h, w, sm_count());
        active_paths[l] = it;  // SOR iterations per solver launch
        variational_level(c, T, lv.I0, lv.I1, sp(S_AVG, w), sp(S_DUN, w), sp(S_DVN, w), h, w, k, P.fixed_point_iterations,
                          P.sor_iterations, it, CLS_SOR, CLS_TERMS, CLS_DERIV, CLS_PYR);
        if (l > 0) {
            const DLevel &nx = L_.levels[l - 1];
            Plane nu = sp(ui ? S_U : S_UN, nx.cols), nv = sp(ui ? S_V : S_VN, nx.cols);
            B2F_LAUNCH(c, CLS_PYR, 2.0 * 4.0 * (npx + (double)nx.rows * nx.cols), k_df_resize,
                       dim3(div_up(nx.cols, 32), div_up(nx.rows, 8), 2), block, 0, T.u, T.v, h, w, nu, nv, nx.rows,
                       nx.cols, (double)w / nx.cols, (double)h / nx.rows, mul, 1);
            ui ^= 1;
        }
    }
    final_ui_ = ui;
}

int DeepFlowEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    if ((I0->type != B2F_8UC1 && I0->type != B2F_32FC1) || I1->type != I0->type) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
    // the engine's pre-smoothing is the 3-tap kernel: kernelLen = floor(3 sigma) * 2 + 1 == 3
    const float sigma_f = static_cast<float>(P.sigma);
    if (!(sigma_f > 0.0f) || static_cast<int>(std::floor(3.0f * sigma_f)) * 2 + 1 != 3 || P.min_size < 0 ||
        P.max_layers < 0 || P.fixed_point_iterations < 0 || P.sor_iterations < 0 || !(P.downscale_factor > 0.0 && P.downscale_factor < 1.0) || !(P.alpha >= 0.0) ||
        !(P.delta >= 0.0) || !(P.gamma >= 0.0) || !(P.omega > 0.0 && P.omega < 2.0))
        return B2F_BAD_ARG;
    const size_t esz = I0->type == B2F_8UC1 ? 1 : 4;
    if (I0->step < (size_t)I0->cols * esz || I1->step < (size_t)I1->cols * esz || !flow_step_ok(flow)) return B2F_BAD_ARG;
    const int rows = I0->rows, cols = I0->cols;
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
    active_paths.assign(L_.levels.size(), 0.0);

    const ImageView vf = flow_view(flow, rows, cols);
    {
        // deepflow.cpp: convertTo(CV_32F) without scaling, then GaussianBlur with getGaussianKernel(3, sigma, CV_32F) --
        // sigma is the reference's float member, widened to double; taps computed in double, normalised, stored as float
        const double sg = static_cast<double>(static_cast<float>(P.sigma)), sc = -0.5 / (sg * sg);
        const double t0 = std::exp(sc), t1 = 1.0, sum = 1.0 / (t0 + t1 + t0);
        const float k0 = static_cast<float>(t1 * sum), k1 = static_cast<float>(t0 * sum);
        const dim3 grid(div_up(cols, 32), div_up(rows, 8), 2), block(32, 8);
        const double bytes = 2.0 * rows * cols * (esz + 4.0);
        const char *p0 = static_cast<const char *>(I0->data), *p1 = static_cast<const char *>(I1->data);
        if (I0->type == B2F_8UC1)
            B2F_LAUNCH(c, CLS_PYR, bytes, k_df_blur<unsigned char>, grid, block, 0, p0, I0->step, p1, I1->step,
                       L_.levels[0].I0, L_.levels[0].I1, rows, cols, k0, k1);
        else
            B2F_LAUNCH(c, CLS_PYR, bytes, k_df_blur<float>, grid, block, 0, p0, I0->step, p1, I1->step, L_.levels[0].I0,
                       L_.levels[0].I1, rows, cols, k0, k1);
    }

    const bool want_graph = knobs.use_graph && !profiling && s != nullptr;
    if (want_graph) {
        graph_.run(*this, c, s, GraphKey{rows, cols, P, L_.levels[0].I0.p}, [&](Ctx &g) { solve(g); });
    } else {
        solve(c);
    }
    merge_flow(c, CLS_PYR, sp(final_ui_ ? S_UN : S_U, cols), sp(final_ui_ ? S_VN : S_V, cols), vf);
    return finish(c, s);
}

int DeepFlowEngine::set_param(int id, double v) {
    switch (id) {
        case B2F_DEEP_SIGMA: P.sigma = v; break;
        case B2F_DEEP_MIN_SIZE: P.min_size = static_cast<int>(v); break;
        case B2F_DEEP_DOWNSCALE_FACTOR: P.downscale_factor = v; break;
        case B2F_DEEP_FIXED_POINT_ITERATIONS: P.fixed_point_iterations = static_cast<int>(v); break;
        case B2F_DEEP_SOR_ITERATIONS: P.sor_iterations = static_cast<int>(v); break;
        case B2F_DEEP_ALPHA: P.alpha = v; break;
        case B2F_DEEP_DELTA: P.delta = v; break;
        case B2F_DEEP_GAMMA: P.gamma = v; break;
        case B2F_DEEP_OMEGA: P.omega = v; break;
        case B2F_DEEP_MAX_LAYERS: P.max_layers = static_cast<int>(v); break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

int DeepFlowEngine::get_param(int id, double *v) const {
    switch (id) {
        case B2F_DEEP_SIGMA: *v = P.sigma; break;
        case B2F_DEEP_MIN_SIZE: *v = P.min_size; break;
        case B2F_DEEP_DOWNSCALE_FACTOR: *v = P.downscale_factor; break;
        case B2F_DEEP_FIXED_POINT_ITERATIONS: *v = P.fixed_point_iterations; break;
        case B2F_DEEP_SOR_ITERATIONS: *v = P.sor_iterations; break;
        case B2F_DEEP_ALPHA: *v = P.alpha; break;
        case B2F_DEEP_DELTA: *v = P.delta; break;
        case B2F_DEEP_GAMMA: *v = P.gamma; break;
        case B2F_DEEP_OMEGA: *v = P.omega; break;
        case B2F_DEEP_MAX_LAYERS: *v = P.max_layers; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

}  // namespace

}  // namespace b2f

extern "C" {

void b2f_deepflow_default_params(b2f_deepflow_params *p) {
    if (!p) return;
    p->sigma = 0.6;
    p->min_size = 25;
    p->downscale_factor = 0.95;
    p->fixed_point_iterations = 5;
    p->sor_iterations = 25;
    p->alpha = 1.0;
    p->delta = 0.5;
    p->gamma = 5.0;
    p->omega = 1.6;
    p->max_layers = 200;
}

int b2f_deepflow_create(const b2f_deepflow_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_deepflow_params d;
    b2f_deepflow_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::DeepFlowEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
