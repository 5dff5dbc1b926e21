// cudaoptflow_compat.hpp -- header-only C++ adapter that reproduces the reference's public API
// for the dense optical-flow path on top of the C ABI (include/b200flow.h).
//
// Reference interface mirrored (modules/cudaoptflow/include/opencv2/cudaoptflow.hpp):
//   DenseOpticalFlow::calc                      :70-81
//   BroxOpticalFlow (+create defaults)          :155-186
//   DensePyrLKOpticalFlow                       :230-250
//   FarnebackOpticalFlow                        :258-294
//   OpticalFlowDual_TVL1                        :305-386
// Same class names, method names, argument order, defaults and getDefaultName() strings, so a
// call site only changes its namespace:   namespace cvcuda = b200flow::cuda;
//
// With OpenCV's core headers on the include path the adapter is expressed in the real
// cv::cuda::GpuMat / cv::cuda::Stream / cv::Ptr / cv::Algorithm types; without them (this repo's
// build container) it uses the field-compatible stand-ins of gpumat_shim.hpp.
#pragma once

#include "../b200flow.h"

#if defined(B200FLOW_WITH_OPENCV) || (defined(__has_include) && __has_include(<opencv2/core/cuda.hpp>))
#include <opencv2/core.hpp>
#include <opencv2/core/cuda.hpp>
#include <opencv2/core/cuda_stream_accessor.hpp>
namespace b200flow {
namespace detail {
using cv::Algorithm;
using cv::InputArray;
using cv::InputOutputArray;
using cv::OutputArray;
using cv::Ptr;
using cv::Size;
using cv::String;
using cv::cuda::GpuMat;
using cv::cuda::Stream;
template <class T, class... A> Ptr<T> make(A &&...a) { return cv::makePtr<T>(std::forward<A>(a)...); }
inline GpuMat in_mat(InputArray a) { return a.getGpuMat(); }
inline GpuMat &out_mat(InputOutputArray a, Size sz, bool keep) {
    if (!keep) a.create(sz, CV_32FC2);
    return a.getGpuMatRef();
}
inline cv::InputOutputArray noArray() { return cv::noArray(); }
inline bool needed(OutputArray a) { return a.needed(); }
// (re)allocate an output like the reference does (getOutputMat / create) and hand back the header
inline GpuMat &out_create(OutputArray a, int rows, int cols, int type) {
    a.create(rows, cols, type);
    return a.getGpuMatRef();
}
inline GpuMat &out_ref(InputOutputArray a) { return a.getGpuMatRef(); }
inline cudaStream_t raw(Stream &s) { return cv::cuda::StreamAccessor::getStream(s); }
[[noreturn]] inline void fail(int status, const char *where) {
    const int code = status == B2F_CUDA_ERROR || status == B2F_OUT_OF_MEMORY ? cv::Error::GpuApiCallError
                     : status == B2F_NO_DEVICE ? cv::Error::GpuNotSupported : cv::Error::StsAssert;
    cv::error(code, b2f_status_string(status), where, __FILE__, __LINE__);
    throw 0;
}
}  // namespace detail
}  // namespace b200flow
#else
#include "gpumat_shim.hpp"
namespace b200flow {
namespace detail {
using namespace shim;
template <class T, class... A> Ptr<T> make(A &&...a) { return shim::makePtr<T>(std::forward<A>(a)...); }
inline const GpuMat &in_mat(InputArray a) { return a; }
inline GpuMat &out_mat(InputOutputArray a, Size sz, bool keep) {
    if (!keep) a.create(sz, CV_32FC2);
    return a;
}
using shim::noArray;
inline bool needed(OutputArray a) { return &a != &shim::noArray(); }
inline GpuMat &out_create(OutputArray a, int rows, int cols, int type) {
    a.create(rows, cols, type);
    return a;
}
inline GpuMat &out_ref(InputOutputArray a) { return a; }
inline cudaStream_t raw(Stream &s) { return s.cudaPtr(); }
[[noreturn]] inline void fail(int status, const char *where) {
    const int code = status == B2F_CUDA_ERROR || status == B2F_OUT_OF_MEMORY ? -217 /*GpuApiCallError*/
                     : status == B2F_NO_DEVICE ? -216 /*GpuNotSupported*/ : -215 /*StsAssert*/;
    throw Exception(code, std::string(where) + ": " + b2f_status_string(status));
}
}  // namespace detail
}  // namespace b200flow
#endif

namespace b200flow {
namespace cuda {

using detail::Algorithm;
using detail::GpuMat;
using detail::InputArray;
using detail::InputOutputArray;
using detail::OutputArray;
using detail::Ptr;
using detail::Size;
using detail::Stream;
using detail::String;

enum { OPTFLOW_USE_INITIAL_FLOW = 4, OPTFLOW_FARNEBACK_GAUSSIAN = 256 };

/** cv::cuda::DenseOpticalFlow (cudaoptflow.hpp:70-81). */
class DenseOpticalFlow : public Algorithm {
public:
    virtual void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) = 0;
};

namespace impl {

// Shared calc(): describe the GpuMats as b2f_images (field-for-field), allocate `flow` the way the
// reference does inside calc (cuda::merge -> getOutputMat, cudaarithm split_merge.cu:130), call b2f_calc.
class HandleOwner {
public:
    ~HandleOwner() { b2f_destroy(h_); }

protected:
    b2f_handle *h_ = nullptr;
    void run(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream, bool reads_flow) {
        const auto &a = detail::in_mat(I0);
        const auto &b = detail::in_mat(I1);
        auto &f = detail::out_mat(flow, a.size(), reads_flow);
        b2f_image i0{a.data, a.step, a.rows, a.cols, a.type()};
        b2f_image i1{b.data, b.step, b.rows, b.cols, b.type()};
        b2f_image fl{f.data, f.step, f.rows, f.cols, f.type()};
        const int st = b2f_calc(h_, &i0, &i1, &fl, detail::raw(stream));
        if (st != B2F_OK) detail::fail(st, "DenseOpticalFlow::calc");
    }
    double get(int id) const {
        double v = 0;
        b2f_get_param(h_, id, &v);
        return v;
    }
    void set(int id, double v) {
        const int st = b2f_set_param(h_, id, v);
        if (st != B2F_OK) detail::fail(st, "set");
    }
};

}  // namespace impl

#define B2F_ACCESSOR(T, Name, ID)                          \
    T get##Name() const { return static_cast<T>(get(ID)); } \
    void set##Name(T v) { set(ID, static_cast<double>(v)); }

/** cv::cuda::OpticalFlowDual_TVL1 (cudaoptflow.hpp:305-386). */
class OpticalFlowDual_TVL1 : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    B2F_ACCESSOR(double, Tau, B2F_TVL1_TAU)
    B2F_ACCESSOR(double, Lambda, B2F_TVL1_LAMBDA)
    B2F_ACCESSOR(double, Gamma, B2F_TVL1_GAMMA)
    B2F_ACCESSOR(double, Theta, B2F_TVL1_THETA)
    B2F_ACCESSOR(int, NumScales, B2F_TVL1_NSCALES)
    B2F_ACCESSOR(int, NumWarps, B2F_TVL1_WARPS)
    B2F_ACCESSOR(double, Epsilon, B2F_TVL1_EPSILON)
    B2F_ACCESSOR(int, NumIterations, B2F_TVL1_ITERATIONS)
    B2F_ACCESSOR(double, ScaleStep, B2F_TVL1_SCALE_STEP)
    B2F_ACCESSOR(bool, UseInitialFlow, B2F_TVL1_USE_INITIAL_FLOW)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, getUseInitialFlow());
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<OpticalFlowDual_TVL1> create(double tau = 0.25, double lambda = 0.15, double theta = 0.3,
                                            int nscales = 5, int warps = 5, double epsilon = 0.01,
                                            int iterations = 300, double scaleStep = 0.8, double gamma = 0.0,
                                            bool useInitialFlow = false) {
        b2f_tvl1_params p{tau, lambda, theta, nscales, warps, epsilon, iterations, scaleStep, gamma, useInitialFlow};
        auto o = detail::make<OpticalFlowDual_TVL1>();
        const int st = b2f_tvl1_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "OpticalFlowDual_TVL1::create");
        return o;
    }
};

/** cv::cuda::FarnebackOpticalFlow (cudaoptflow.hpp:258-294). */
class FarnebackOpticalFlow : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    B2F_ACCESSOR(int, NumLevels, B2F_FARN_NUM_LEVELS)
    B2F_ACCESSOR(double, PyrScale, B2F_FARN_PYR_SCALE)
    B2F_ACCESSOR(bool, FastPyramids, B2F_FARN_FAST_PYRAMIDS)
    B2F_ACCESSOR(int, WinSize, B2F_FARN_WIN_SIZE)
    B2F_ACCESSOR(int, NumIters, B2F_FARN_NUM_ITERS)
    B2F_ACCESSOR(int, PolyN, B2F_FARN_POLY_N)
    B2F_ACCESSOR(double, PolySigma, B2F_FARN_POLY_SIGMA)
    B2F_ACCESSOR(int, Flags, B2F_FARN_FLAGS)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, (getFlags() & OPTFLOW_USE_INITIAL_FLOW) != 0);
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<FarnebackOpticalFlow> create(int numLevels = 5, double pyrScale = 0.5, bool fastPyramids = false,
                                            int winSize = 13, int numIters = 10, int polyN = 5,
                                            double polySigma = 1.1, int flags = 0) {
        b2f_farneback_params p{numLevels, pyrScale, fastPyramids, winSize, numIters, polyN, polySigma, flags};
        auto o = detail::make<FarnebackOpticalFlow>();
        const int st = b2f_farneback_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "FarnebackOpticalFlow::create");
        return o;
    }
};

/** cv::cuda::BroxOpticalFlow (cudaoptflow.hpp:155-186). */
class BroxOpticalFlow : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    B2F_ACCESSOR(double, FlowSmoothness, B2F_BROX_ALPHA)
    B2F_ACCESSOR(double, GradientConstancyImportance, B2F_BROX_GAMMA)
    B2F_ACCESSOR(double, PyramidScaleFactor, B2F_BROX_SCALE_FACTOR)
    B2F_ACCESSOR(int, InnerIterations, B2F_BROX_INNER_ITERATIONS)
    B2F_ACCESSOR(int, OuterIterations, B2F_BROX_OUTER_ITERATIONS)
    B2F_ACCESSOR(int, SolverIterations, B2F_BROX_SOLVER_ITERATIONS)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, false);
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<BroxOpticalFlow> create(double alpha = 0.197, double gamma = 50.0, double scale_factor = 0.8,
                                       int inner_iterations = 5, int outer_iterations = 150,
                                       int solver_iterations = 10) {
        b2f_brox_params p{alpha, gamma, scale_factor, inner_iterations, outer_iterations, solver_iterations};
        auto o = detail::make<BroxOpticalFlow>();
        const int st = b2f_brox_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "BroxOpticalFlow::create");
        return o;
    }
};

/** cv::cuda::DensePyrLKOpticalFlow (cudaoptflow.hpp:230-250). */
class DensePyrLKOpticalFlow : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    Size getWinSize() const { return Size((int)get(B2F_LK_WIN_WIDTH), (int)get(B2F_LK_WIN_HEIGHT)); }
    void setWinSize(Size s) {
        set(B2F_LK_WIN_WIDTH, s.width);
        set(B2F_LK_WIN_HEIGHT, s.height);
    }
    B2F_ACCESSOR(int, MaxLevel, B2F_LK_MAX_LEVEL)
    B2F_ACCESSOR(int, NumIters, B2F_LK_ITERS)
    B2F_ACCESSOR(bool, UseInitialFlow, B2F_LK_USE_INITIAL_FLOW)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, getUseInitialFlow());
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<DensePyrLKOpticalFlow> create(Size winSize = Size(13, 13), int maxLevel = 3, int iters = 30,
                                             bool useInitialFlow = false) {
        b2f_denselk_params p{winSize.width, winSize.height, maxLevel, iters, useInitialFlow};
        auto o = detail::make<DensePyrLKOpticalFlow>();
        const int st = b2f_denselk_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "DensePyrLKOpticalFlow::create");
        return o;
    }
};

/** cv::optflow::createOptFlow_DeepFlow (optflow.hpp; modules/optflow/src/deepflow.cpp) on the GPU.  The reference's
 *  OpticalFlowDeepFlow is a CPU cv::DenseOpticalFlow with no accessors; this class takes the cv::cuda calling convention
 *  (device images and a Stream) and names its accessors after the constructor's fields.  `flow` is written, never
 *  read. */
class DeepFlowOpticalFlow : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    B2F_ACCESSOR(double, Sigma, B2F_DEEP_SIGMA)
    B2F_ACCESSOR(int, MinSize, B2F_DEEP_MIN_SIZE)
    B2F_ACCESSOR(double, DownscaleFactor, B2F_DEEP_DOWNSCALE_FACTOR)
    B2F_ACCESSOR(int, FixedPointIterations, B2F_DEEP_FIXED_POINT_ITERATIONS)
    B2F_ACCESSOR(int, SorIterations, B2F_DEEP_SOR_ITERATIONS)
    B2F_ACCESSOR(double, Alpha, B2F_DEEP_ALPHA)
    B2F_ACCESSOR(double, Delta, B2F_DEEP_DELTA)
    B2F_ACCESSOR(double, Gamma, B2F_DEEP_GAMMA)
    B2F_ACCESSOR(double, Omega, B2F_DEEP_OMEGA)
    B2F_ACCESSOR(int, MaxLayers, B2F_DEEP_MAX_LAYERS)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, false);
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<DeepFlowOpticalFlow> create(double sigma = 0.6, int minSize = 25, double downscaleFactor = 0.95,
                                           int fixedPointIterations = 5, int sorIterations = 25, double alpha = 1.0,
                                           double delta = 0.5, double gamma = 5.0, double omega = 1.6,
                                           int maxLayers = 200) {
        b2f_deepflow_params p{sigma, minSize, downscaleFactor, fixedPointIterations, sorIterations, alpha, delta, gamma,
                              omega, maxLayers};
        auto o = detail::make<DeepFlowOpticalFlow>();
        const int st = b2f_deepflow_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "DeepFlowOpticalFlow::create");
        return o;
    }
};

/** cv::optflow::createOptFlow_DeepFlow with the reference's defaults. */
inline Ptr<DeepFlowOpticalFlow> createOptFlow_DeepFlow() { return DeepFlowOpticalFlow::create(); }

/** cv::DISOpticalFlow (opencv's video module) on the GPU, with its accessors, in the cv::cuda calling convention.  u8
 *  images; with UseInitialFlow `flow` is read as the initial flow (see b2f_dis_params).  Spatial propagation follows OpenCV's OpenCL kernels (see b2f_dis_params). */
class DISOpticalFlow : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    enum { PRESET_ULTRAFAST = B2F_DIS_PRESET_ULTRAFAST, PRESET_FAST = B2F_DIS_PRESET_FAST, PRESET_MEDIUM = B2F_DIS_PRESET_MEDIUM };
    B2F_ACCESSOR(int, FinestScale, B2F_DIS_FINEST_SCALE)
    B2F_ACCESSOR(int, CoarsestScale, B2F_DIS_COARSEST_SCALE)
    B2F_ACCESSOR(int, PatchSize, B2F_DIS_PATCH_SIZE)
    B2F_ACCESSOR(int, PatchStride, B2F_DIS_PATCH_STRIDE)
    B2F_ACCESSOR(int, GradientDescentIterations, B2F_DIS_GRADIENT_DESCENT_ITERATIONS)
    B2F_ACCESSOR(int, VariationalRefinementIterations, B2F_DIS_VARIATIONAL_REFINEMENT_ITERATIONS)
    B2F_ACCESSOR(float, VariationalRefinementAlpha, B2F_DIS_VARIATIONAL_REFINEMENT_ALPHA)
    B2F_ACCESSOR(float, VariationalRefinementDelta, B2F_DIS_VARIATIONAL_REFINEMENT_DELTA)
    B2F_ACCESSOR(float, VariationalRefinementGamma, B2F_DIS_VARIATIONAL_REFINEMENT_GAMMA)
    B2F_ACCESSOR(float, VariationalRefinementEpsilon, B2F_DIS_VARIATIONAL_REFINEMENT_EPSILON)
    B2F_ACCESSOR(bool, UseMeanNormalization, B2F_DIS_USE_MEAN_NORMALIZATION)
    B2F_ACCESSOR(bool, UseSpatialPropagation, B2F_DIS_USE_SPATIAL_PROPAGATION)
    B2F_ACCESSOR(bool, UseInitialFlow, B2F_DIS_USE_INITIAL_FLOW)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, getUseInitialFlow());
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<DISOpticalFlow> create(int preset = PRESET_FAST) {
        b2f_dis_params p;
        b2f_dis_default_params(&p, preset);
        auto o = detail::make<DISOpticalFlow>();
        const int st = b2f_dis_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "DISOpticalFlow::create");
        return o;
    }
};

/** cv::VariationalRefinement (opencv's video module) on the GPU, with its accessors, in the cv::cuda calling convention:
 *  calc refines `flow` (32FC2 of the frame's size, always read) in place, calcUV the same on two 32FC1 planes.  u8 or
 *  float images, used without scaling (see b2f_varref_params). */
class VariationalRefinement : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    B2F_ACCESSOR(int, FixedPointIterations, B2F_VR_FIXED_POINT_ITERATIONS)
    B2F_ACCESSOR(int, SorIterations, B2F_VR_SOR_ITERATIONS)
    B2F_ACCESSOR(float, Omega, B2F_VR_OMEGA)
    B2F_ACCESSOR(float, Alpha, B2F_VR_ALPHA)
    B2F_ACCESSOR(float, Delta, B2F_VR_DELTA)
    B2F_ACCESSOR(float, Gamma, B2F_VR_GAMMA)
    B2F_ACCESSOR(float, Epsilon, B2F_VR_EPSILON)

    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, true);
    }
    void calcUV(InputArray I0, InputArray I1, InputOutputArray flow_u, InputOutputArray flow_v,
                Stream &stream = Stream::Null()) {
        const auto &a = detail::in_mat(I0);
        const auto &b = detail::in_mat(I1);
        auto &u = detail::out_ref(flow_u);
        auto &v = detail::out_ref(flow_v);
        b2f_image i0{a.data, a.step, a.rows, a.cols, a.type()};
        b2f_image i1{b.data, b.step, b.rows, b.cols, b.type()};
        b2f_image iu{u.data, u.step, u.rows, u.cols, u.type()};
        b2f_image iv{v.data, v.step, v.rows, v.cols, v.type()};
        const int st = b2f_calc_uv(h_, &i0, &i1, &iu, &iv, detail::raw(stream));
        if (st != B2F_OK) detail::fail(st, "VariationalRefinement::calcUV");
    }
    String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<VariationalRefinement> create() {
        auto o = detail::make<VariationalRefinement>();
        const int st = b2f_varref_create(nullptr, &o->h_);
        if (st != B2F_OK) detail::fail(st, "VariationalRefinement::create");
        return o;
    }
};

/** cv::cuda::FastOpticalFlowBM (cudalegacy.hpp:202-211): operator() with the reference's signature; flowx / flowy are
 *  (re)allocated as CV_32FC1 of the frame's size.  Also a DenseOpticalFlow (calc writes CV_32FC2 with the handle's
 *  windows).  Refused windows: see b2f_fastbm_params. */
class FastOpticalFlowBM : public DenseOpticalFlow, protected impl::HandleOwner {
public:
    FastOpticalFlowBM() {
        const int st = b2f_fastbm_create(nullptr, &h_);
        if (st != B2F_OK) detail::fail(st, "FastOpticalFlowBM");
    }
    B2F_ACCESSOR(int, SearchWindow, B2F_FBM_SEARCH_WINDOW)
    B2F_ACCESSOR(int, BlockWindow, B2F_FBM_BLOCK_WINDOW)

    void operator()(const GpuMat &I0, const GpuMat &I1, GpuMat &flowx, GpuMat &flowy, int search_window = 21,
                    int block_window = 7, Stream &stream = Stream::Null()) {
        setSearchWindow(search_window);
        setBlockWindow(block_window);
        flowx.create(I0.rows, I0.cols, 5 /*CV_32FC1*/);
        flowy.create(I0.rows, I0.cols, 5 /*CV_32FC1*/);
        b2f_image i0{I0.data, I0.step, I0.rows, I0.cols, I0.type()};
        b2f_image i1{I1.data, I1.step, I1.rows, I1.cols, I1.type()};
        b2f_image u{flowx.data, flowx.step, flowx.rows, flowx.cols, flowx.type()};
        b2f_image v{flowy.data, flowy.step, flowy.rows, flowy.cols, flowy.type()};
        const int st = b2f_calc_uv(h_, &i0, &i1, &u, &v, detail::raw(stream));
        if (st != B2F_OK) detail::fail(st, "FastOpticalFlowBM::operator()");
    }
    void calc(InputArray I0, InputArray I1, InputOutputArray flow, Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, false);
    }
    String getDefaultName() const override { return b2f_default_name(h_); }
};

/** cv::cuda::calcOpticalFlowBM (cudalegacy.hpp:196-200), the reference's signature.  velx / vely are (re)allocated as
 *  CV_32FC1 of velSize unless use_previous is set, when they are read first and must already be of velSize.  `buf` is
 *  accepted and left untouched: the spiral table is computed on the device. */
inline void calcOpticalFlowBM(const GpuMat &prev, const GpuMat &curr, Size block_size, Size shift_size, Size max_range,
                              bool use_previous, GpuMat &velx, GpuMat &vely, GpuMat &buf, Stream &stream = Stream::Null()) {
    (void)buf;
    int vr = 0, vc = 0;
    int st = b2f_calc_optical_flow_bm_size(prev.rows, prev.cols, block_size.width, block_size.height, shift_size.width,
                                           shift_size.height, max_range.width, max_range.height, &vr, &vc, nullptr);
    if (st != B2F_OK) detail::fail(st, "calcOpticalFlowBM");
    if (!use_previous) {
        velx.create(vr, vc, 5 /*CV_32FC1*/);
        vely.create(vr, vc, 5 /*CV_32FC1*/);
    }
    b2f_image p{prev.data, prev.step, prev.rows, prev.cols, prev.type()};
    b2f_image c{curr.data, curr.step, curr.rows, curr.cols, curr.type()};
    b2f_image x{velx.data, velx.step, velx.rows, velx.cols, velx.type()};
    b2f_image y{vely.data, vely.step, vely.rows, vely.cols, vely.type()};
    st = b2f_calc_optical_flow_bm(&p, &c, block_size.width, block_size.height, shift_size.width, shift_size.height,
                                  max_range.width, max_range.height, use_previous ? 1 : 0, &x, &y, detail::raw(stream));
    if (st != B2F_OK) detail::fail(st, "calcOpticalFlowBM");
}

#undef B2F_ACCESSOR

/** cv::cuda::SparsePyrLKOpticalFlow (cudaoptflow.hpp:189-226), same signature as the reference's
 *  SparseOpticalFlow::calc (:99-103): prevPts / nextPts are 1 x N CV_32FC2, status 1 x N CV_8UC1, err 1 x N CV_32FC1
 *  and optional (`= cv::noArray()`); nextPts, status and err are (re)allocated like the reference does
 *  (pyrlk.cpp:165,172,176). */
class SparsePyrLKOpticalFlow : public Algorithm {
public:
    ~SparsePyrLKOpticalFlow() { b2f_sparselk_destroy(h_); }
    void calc(InputArray prevImg_, InputArray nextImg_, InputArray prevPts_, InputOutputArray nextPts_, OutputArray status_,
              OutputArray err_ = detail::noArray(), Stream &stream = Stream::Null()) {
        const auto &prevImg = detail::in_mat(prevImg_);
        const auto &nextImg = detail::in_mat(nextImg_);
        const auto &prevPts = detail::in_mat(prevPts_);
        if (prevPts.cols == 0) return;
        if (prevPts.rows != 1 || prevPts.type() != 13 /*CV_32FC2*/) detail::fail(B2F_BAD_ARG, "SparsePyrLKOpticalFlow::calc");
        GpuMat *nextPts = &detail::out_ref(nextPts_);
        if (!getUseInitialFlow()) nextPts = &detail::out_create(nextPts_, 1, prevPts.cols, 13);
        else if (nextPts->cols != prevPts.cols || nextPts->type() != 13) detail::fail(B2F_SIZE_MISMATCH, "SparsePyrLKOpticalFlow::calc");
        GpuMat &status = detail::out_create(status_, 1, prevPts.cols, 0 /*CV_8UC1*/);
        GpuMat *err = detail::needed(err_) ? &detail::out_create(err_, 1, prevPts.cols, 5 /*CV_32FC1*/) : nullptr;
        b2f_image i0{prevImg.data, prevImg.step, prevImg.rows, prevImg.cols, prevImg.type()};
        b2f_image i1{nextImg.data, nextImg.step, nextImg.rows, nextImg.cols, nextImg.type()};
        const int st = b2f_sparselk_calc(h_, &i0, &i1, reinterpret_cast<const float *>(prevPts.data),
                                         reinterpret_cast<float *>(nextPts->data), reinterpret_cast<unsigned char *>(status.data),
                                         err ? reinterpret_cast<float *>(err->data) : nullptr, prevPts.cols, detail::raw(stream));
        if (st != B2F_OK) detail::fail(st, "SparsePyrLKOpticalFlow::calc");
    }
    /** round-1 spelling: `err` as a pointer (nullptr = cv::noArray()) */
    void calc(InputArray prevImg, InputArray nextImg, InputArray prevPts, InputOutputArray nextPts, OutputArray status,
              GpuMat *err, Stream &stream = Stream::Null()) {
        if (err) calc(prevImg, nextImg, prevPts, nextPts, status, *err, stream);
        else calc(prevImg, nextImg, prevPts, nextPts, status, detail::noArray(), stream);
    }
    Size getWinSize() const { const auto p = params(); return Size(p.win_width, p.win_height); }
    void setWinSize(Size s) { auto p = params(); p.win_width = s.width; p.win_height = s.height; b2f_sparselk_set_params(h_, &p); }
    int getMaxLevel() const { return params().max_level; }
    void setMaxLevel(int v) { auto p = params(); p.max_level = v; b2f_sparselk_set_params(h_, &p); }
    int getNumIters() const { return params().iters; }
    void setNumIters(int v) { auto p = params(); p.iters = v; b2f_sparselk_set_params(h_, &p); }
    bool getUseInitialFlow() const { return params().use_initial_flow != 0; }
    void setUseInitialFlow(bool v) { auto p = params(); p.use_initial_flow = v; b2f_sparselk_set_params(h_, &p); }
    String getDefaultName() const override { return "SparseOpticalFlow.SparsePyrLKOpticalFlow"; }

    static Ptr<SparsePyrLKOpticalFlow> create(Size winSize = Size(21, 21), int maxLevel = 3, int iters = 30,
                                              bool useInitialFlow = false) {
        b2f_sparselk_params p{winSize.width, winSize.height, maxLevel, iters, useInitialFlow};
        auto o = detail::make<SparsePyrLKOpticalFlow>();
        const int st = b2f_sparselk_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "SparsePyrLKOpticalFlow::create");
        return o;
    }

private:
    b2f_sparse *h_ = nullptr;
    b2f_sparselk_params params() const {
        b2f_sparselk_params p{};
        b2f_sparselk_get_params(h_, &p);
        return p;
    }
};

/** cv::cuda::interpolateFrames (cudalegacy.hpp:229, src/interpolate_frames.cpp:54-111): same argument order;
 *  newFrame and buf are (re)allocated like the reference does (:64-67).  `corrected` = false keeps the
 *  reference's behaviour including its defects (see b200flow.h). */
inline void interpolateFrames(const GpuMat &frame0, const GpuMat &frame1, const GpuMat &fu, const GpuMat &fv,
                              const GpuMat &bu, const GpuMat &bv, float pos, GpuMat &newFrame, GpuMat &buf,
                              Stream &stream = Stream::Null(), bool corrected = false) {
    newFrame.create(frame0.rows, frame0.cols, frame0.type());
    buf.create(6 * frame0.rows, frame0.cols, frame0.type());
    auto img = [](const GpuMat &m) { return b2f_image{m.data, m.step, m.rows, m.cols, m.type()}; };
    b2f_image f0 = img(frame0), f1 = img(frame1), iu = img(fu), iv = img(fv), ju = img(bu), jv = img(bv);
    b2f_image out = img(newFrame), scratch = img(buf);
    const int st = b2f_interpolate_frames(&f0, &f1, &iu, &iv, &ju, &jv, pos, &out, &scratch,
                                          corrected ? B2F_INTERP_CORRECTED : B2F_INTERP_REFERENCE, detail::raw(stream));
    if (st != B2F_OK) detail::fail(st, "interpolateFrames");
}

}  // namespace cuda
}  // namespace b200flow
