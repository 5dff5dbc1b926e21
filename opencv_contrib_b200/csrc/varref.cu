// varref.cu -- cv::VariationalRefinement (opencv's video module) for sm_90a: the caller's flow refined in place.
//
// One calcUV call: both frames converted to float (no scaling), the flow split into planes, one level of the
// variational solver DeepFlow and DIS run (variational.cuh) with this handle's alpha, delta, gamma, epsilon and omega,
// and the result merged back into the caller's buffer.  oracle/dis_model.py refine states what it computes; this file is
// compiled with -fmad=false (csrc/Makefile), so the float model follows the engine bit for bit.
//
// Per call: conversion (1 launch) and split (1), then, inside the handle's CUDA graph, warp (1) + derivatives (1), per
// fixed-point step one system-terms launch and ceil(sor / k) solver launches, and the add (1); last the merge (1).  A
// frame that fits one 64x64 region runs its fixed-point steps in one single-CTA launch.
//
// Kernel classes: 0 sor (44 B/px algorithmic per SOR iteration), 1 system terms (88 B/px), 2 warp + derivatives,
// 3 conversion, split, add and merge.
#include "variational.cuh"

#include <new>

namespace b2f {

namespace {

static bool same_params(const b2f_varref_params &a, const b2f_varref_params &b) {
    return a.fixed_point_iterations == b.fixed_point_iterations && a.sor_iterations == b.sor_iterations &&
           a.omega == b.omega && a.alpha == b.alpha && a.delta == b.delta && a.gamma == b.gamma &&
           a.epsilon == b.epsilon;
}

class VarRefEngine : public b2f_handle {
public:
    explicit VarRefEngine(const b2f_varref_params &p) : P(p) { algo = ALGO_VARREF; }
    b2f_varref_params P;

    int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) override;
    int set_param(int id, double v) override;
    int get_param(int id, double *v) const override;
    // what cv2.VariationalRefinement reports: the class does not override getDefaultName
    const char *default_name() const override { return "my_object"; }
    bool reads_flow() const override { return true; }
    const char *class_name(int cls) const override {
        static const char *n[] = {"varref_sor", "varref_terms", "varref_warp_derivatives", "varref_io"};
        return (cls >= 0 && cls < 4) ? n[cls] : "";
    }
    size_t workspace_bytes(int rows, int cols, int type) override {
        (void)type;
        Layout L;
        return layout(rows, cols, true, L);
    }

private:
    // the average of I0 and the warped I1 (S_AVG) is dead once the derivatives are written: it shares A12's plane
    enum { S_I0 = 0, S_I1, S_IX, S_IY, S_IZ, S_IXX, S_IXY, S_IYY, S_IXZ, S_IYZ, S_U, S_V, S_DU, S_DV, S_DUN, S_DVN,
           S_A12, S_B1, S_B2, S_DENU, S_DENV, S_WR, S_WD, S_COUNT, S_AVG = S_A12 };
    struct Layout {
        int rows = 0, cols = 0;
        float *planes[S_COUNT] = {};
    };
    Layout L_;
    struct GraphKey {  // the schedule reads no knob
        int rows, cols;
        b2f_varref_params P;
        const void *base;
        bool operator==(const GraphKey &o) const {
            return rows == o.rows && cols == o.cols && same_params(P, o.P) && base == o.base;
        }
    };
    GraphCache<GraphKey> graph_;

    size_t layout(int rows, int cols, bool counting, Layout &L);
    cudaError_t ensure_workspace(int rows, int cols);
    Plane sp(int idx) const { return Plane{L_.planes[idx], plane_pitch(L_.cols)}; }
    void solve(Ctx &c);
};

size_t VarRefEngine::layout(int rows, int cols, bool counting, Layout &L) {
    Arena tmp;
    Arena &A = counting ? tmp : arena;
    A.begin(counting);
    L.rows = rows;
    L.cols = cols;
    for (int i = 0; i < S_COUNT; ++i) L.planes[i] = A.plane(rows, cols).p;
    return A.used();
}

cudaError_t VarRefEngine::ensure_workspace(int rows, int cols) {
    if (L_.rows == rows && L_.cols == cols && arena.capacity() > 0) return cudaSuccess;
    Layout tmp;
    const size_t need = layout(rows, cols, true, tmp);
    graph_.destroy();
    cudaError_t e = arena.reserve(need);
    if (e != cudaSuccess) return e;
    layout(rows, cols, false, L_);
    return cudaSuccess;
}

void VarRefEngine::solve(Ctx &c) {
    const int h = L_.rows, w = L_.cols;
    // cv2 accepts any count; a count below one runs no step
    const int fp = std::max(0, P.fixed_point_iterations), sor = std::max(0, P.sor_iterations);
    // the VariationalRefinement members as DIS sets them (dis.cu): halves of alpha, delta and gamma, epsilon squared
    DFParams k;
    k.alpha2 = static_cast<float>(P.alpha) * 0.5f;
    k.delta2 = static_cast<float>(P.delta) * 0.5f;
    k.gamma2 = static_cast<float>(P.gamma) * 0.5f;
    k.z2 = ZETA * ZETA;
    k.e2 = static_cast<float>(P.epsilon) * static_cast<float>(P.epsilon);
    k.omega = static_cast<float>(P.omega);
    k.omo = 1.0f - k.omega;
    LevelPlanes T;
    T.Ix = sp(S_IX); T.Iy = sp(S_IY); T.Iz = sp(S_IZ);
    T.Ixx = sp(S_IXX); T.Ixy = sp(S_IXY); T.Iyy = sp(S_IYY); T.Ixz = sp(S_IXZ); T.Iyz = sp(S_IYZ);
    T.u = sp(S_U); T.v = sp(S_V);
    T.du = sp(S_DU); T.dv = sp(S_DV);
    T.a12 = sp(S_A12); T.b1 = sp(S_B1); T.b2 = sp(S_B2);
    T.den_u = sp(S_DENU); T.den_v = sp(S_DENV); T.wr = sp(S_WR); T.wd = sp(S_WD);
    const int it = variational_iters_per_launch(sor, h, w, sm_count());
    active_paths[0] = fp > 0 && sor > 0 ? it : 0;  // SOR iterations per solver launch
    variational_level(c, T, sp(S_I0), sp(S_I1), sp(S_AVG), sp(S_DUN), sp(S_DVN), h, w, k, fp, sor, it, CLS_SOR, CLS_TERMS,
                      CLS_DERIV, CLS_PYR);
}

int VarRefEngine::calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) {
    if ((I0->type != B2F_8UC1 && I0->type != B2F_32FC1) || I1->type != I0->type) return B2F_UNSUPPORTED_TYPE;
    if (I0->rows != I1->rows || I0->cols != I1->cols) return B2F_SIZE_MISMATCH;
    if (!flow_type_ok(flow)) return B2F_UNSUPPORTED_TYPE;
    if (flow->rows != I0->rows || flow->cols != I0->cols) return B2F_SIZE_MISMATCH;
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
    stats.levels = 1;
    stats.iterations_run = 0;
    active_paths.assign(1, 0.0);

    // the caller's images and flow are read before the graph, which must not bake their addresses in
    const ImageView a{I0->data, I0->step, rows, cols, I0->type}, b{I1->data, I1->step, rows, cols, I1->type};
    convert_pair(c, CLS_PYR, a, b, sp(S_I0), sp(S_I1), 1.0f);
    const ImageView vf = flow_view(flow, rows, cols);
    split_flow(c, CLS_PYR, vf, sp(S_U), sp(S_V));
    const bool want_graph = knobs.use_graph && !profiling && s != nullptr;
    if (want_graph) {
        graph_.run(*this, c, s, GraphKey{rows, cols, P, L_.planes[0]}, [&](Ctx &g) { solve(g); });
    } else {
        solve(c);
    }
    merge_flow(c, CLS_PYR, sp(S_U), sp(S_V), vf);
    return finish(c, s);
}

int VarRefEngine::set_param(int id, double v) {
    switch (id) {
        case B2F_VR_FIXED_POINT_ITERATIONS: P.fixed_point_iterations = static_cast<int>(v); break;
        case B2F_VR_SOR_ITERATIONS: P.sor_iterations = static_cast<int>(v); break;
        case B2F_VR_OMEGA: P.omega = v; break;
        case B2F_VR_ALPHA: P.alpha = v; break;
        case B2F_VR_DELTA: P.delta = v; break;
        case B2F_VR_GAMMA: P.gamma = v; break;
        case B2F_VR_EPSILON: P.epsilon = v; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

int VarRefEngine::get_param(int id, double *v) const {
    switch (id) {
        case B2F_VR_FIXED_POINT_ITERATIONS: *v = P.fixed_point_iterations; break;
        case B2F_VR_SOR_ITERATIONS: *v = P.sor_iterations; break;
        case B2F_VR_OMEGA: *v = P.omega; break;
        case B2F_VR_ALPHA: *v = P.alpha; break;
        case B2F_VR_DELTA: *v = P.delta; break;
        case B2F_VR_GAMMA: *v = P.gamma; break;
        case B2F_VR_EPSILON: *v = P.epsilon; break;
        default: return B2F_BAD_ARG;
    }
    return B2F_OK;
}

}  // namespace

}  // namespace b2f

extern "C" {

void b2f_varref_default_params(b2f_varref_params *p) {
    if (!p) return;
    p->fixed_point_iterations = 5;
    p->sor_iterations = 5;
    p->omega = 1.6;
    p->alpha = 20.0;
    p->delta = 5.0;
    p->gamma = 10.0;
    p->epsilon = 0.001;
}

int b2f_varref_create(const b2f_varref_params *p, b2f_handle **out) {
    if (!out) return B2F_BAD_ARG;
    b2f_varref_params d;
    b2f_varref_default_params(&d);
    if (p) d = *p;
    *out = new (std::nothrow) b2f::VarRefEngine(d);
    return *out ? B2F_OK : B2F_OUT_OF_MEMORY;
}

}  // extern "C"
