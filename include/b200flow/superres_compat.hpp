// superres_compat.hpp -- header-only C++ adapter reproducing the reference's CUDA super-resolution API on top of the C
// ABI (b2f_superres_*, b2f_calc_ext in include/b200flow.h).
//
// Reference interface mirrored (modules/superres/include/opencv2/superres.hpp, superres/optical_flow.hpp):
//   FrameSource                                   superres.hpp:66-73
//   SuperResolution, createSuperResolution_BTVL1_CUDA   :87-200
//   DenseOpticalFlowExt and the four CUDA wrappers      optical_flow.hpp:52-196
// Same class names, method names and argument order, so a call site only changes its namespace:
//   namespace sr = b200flow::superres;
// Frames are GpuMats of 8UC1, 8UC3 or 8UC4.  A DenseOpticalFlowExt that is not one of the four wrappers (the reference
// perf test's ZeroOpticalFlow, for instance) is called for the flows and its planar (u, v) are pushed to the library.
#pragma once

#include "cudaoptflow_compat.hpp"

namespace b200flow {
namespace superres {

using detail::Algorithm;
using detail::GpuMat;
using detail::InputArray;
using detail::OutputArray;
using detail::Ptr;
using detail::Stream;
using detail::String;

/** cv::superres::FrameSource (superres.hpp:66-73). */
class FrameSource {
public:
    virtual ~FrameSource() {}
    virtual void nextFrame(OutputArray frame) = 0;
    virtual void reset() = 0;
};

/** cv::superres::DenseOpticalFlowExt (optical_flow.hpp:52-61). */
class DenseOpticalFlowExt : public Algorithm {
public:
    virtual void calc(InputArray frame0, InputArray frame1, OutputArray flow1, OutputArray flow2 = detail::noArray()) = 0;
    virtual void collectGarbage() = 0;
    // the engine behind one of the four CUDA wrappers; NULL for a caller's own flow
    virtual b2f_handle *engine() const { return nullptr; }
};

#define B2F_EXT_ACCESSOR(T, Name, ID)                      \
    T get##Name() const { return static_cast<T>(get(ID)); } \
    void set##Name(T v) { set(ID, static_cast<double>(v)); }

namespace impl {

inline b2f_image image(const GpuMat &m) { return b2f_image{m.data, m.step, m.rows, m.cols, m.type()}; }

// GpuOpticalFlow (superres/src/optical_flow.cpp:440-497) over one engine handle
class WrapperBase : public DenseOpticalFlowExt {
public:
    ~WrapperBase() override { b2f_destroy(h_); }
    void calc(InputArray frame0, InputArray frame1, OutputArray flow1, OutputArray flow2 = detail::noArray()) override {
        const auto &a = detail::in_mat(frame0);
        const auto &b = detail::in_mat(frame1);
        b2f_image i0 = image(a), i1 = image(b);
        int st;
        if (detail::needed(flow2)) {
            auto &u = detail::out_create(flow1, a.rows, a.cols, B2F_32FC1);
            auto &v = detail::out_create(flow2, a.rows, a.cols, B2F_32FC1);
            b2f_image iu = image(u), iv = image(v);
            st = b2f_calc_ext(h_, &i0, &i1, &iu, &iv, nullptr);
        } else {
            auto &f = detail::out_create(flow1, a.rows, a.cols, B2F_32FC2);
            b2f_image fl = image(f);
            st = b2f_calc_ext(h_, &i0, &i1, &fl, nullptr, nullptr);
        }
        if (st != B2F_OK) detail::fail(st, "DenseOpticalFlowExt::calc");
    }
    void collectGarbage() override {}
    b2f_handle *engine() const override { return h_; }

protected:
    b2f_handle *h_ = nullptr;
    double get(int id) const {
        double v = 0;
        b2f_get_param(h_, id, &v);
        return v;
    }
    void set(int id, double v) {
        const int st = b2f_set_param(h_, id, v);
        if (st != B2F_OK) detail::fail(st, "set");
    }
    void own(int st, const char *where) {
        if (st != B2F_OK) detail::fail(st, where);
    }
};

}  // namespace impl

/** cv::superres::FarnebackOpticalFlow (optical_flow.hpp:64-98), createOptFlow_Farneback_CUDA. */
class FarnebackOpticalFlow : public impl::WrapperBase {
public:
    B2F_EXT_ACCESSOR(double, PyrScale, B2F_FARN_PYR_SCALE)
    B2F_EXT_ACCESSOR(int, LevelsNumber, B2F_FARN_NUM_LEVELS)
    B2F_EXT_ACCESSOR(int, WindowSize, B2F_FARN_WIN_SIZE)
    B2F_EXT_ACCESSOR(int, Iterations, B2F_FARN_NUM_ITERS)
    B2F_EXT_ACCESSOR(int, PolyN, B2F_FARN_POLY_N)
    B2F_EXT_ACCESSOR(double, PolySigma, B2F_FARN_POLY_SIGMA)
    B2F_EXT_ACCESSOR(int, Flags, B2F_FARN_FLAGS)
    FarnebackOpticalFlow() { own(b2f_farneback_create(nullptr, &h_), "createOptFlow_Farneback_CUDA"); }
};

/** cv::superres::DualTVL1OpticalFlow (optical_flow.hpp:103-140), createOptFlow_DualTVL1_CUDA. */
class DualTVL1OpticalFlow : public impl::WrapperBase {
public:
    B2F_EXT_ACCESSOR(double, Tau, B2F_TVL1_TAU)
    B2F_EXT_ACCESSOR(double, Lambda, B2F_TVL1_LAMBDA)
    B2F_EXT_ACCESSOR(double, Theta, B2F_TVL1_THETA)
    B2F_EXT_ACCESSOR(int, ScalesNumber, B2F_TVL1_NSCALES)
    B2F_EXT_ACCESSOR(int, WarpingsNumber, B2F_TVL1_WARPS)
    B2F_EXT_ACCESSOR(double, Epsilon, B2F_TVL1_EPSILON)
    B2F_EXT_ACCESSOR(int, Iterations, B2F_TVL1_ITERATIONS)
    B2F_EXT_ACCESSOR(bool, UseInitialFlow, B2F_TVL1_USE_INITIAL_FLOW)
    DualTVL1OpticalFlow() { own(b2f_tvl1_create(nullptr, &h_), "createOptFlow_DualTVL1_CUDA"); }
};

/** cv::superres::BroxOpticalFlow (optical_flow.hpp:143-178), createOptFlow_Brox_CUDA: the engine is created with
 *  (0.197f, 50.0f, 0.8f, 10, 77, 10) (superres/src/optical_flow.cpp:533). */
class BroxOpticalFlow : public impl::WrapperBase {
public:
    B2F_EXT_ACCESSOR(double, Alpha, B2F_BROX_ALPHA)
    B2F_EXT_ACCESSOR(double, Gamma, B2F_BROX_GAMMA)
    B2F_EXT_ACCESSOR(double, ScaleFactor, B2F_BROX_SCALE_FACTOR)
    B2F_EXT_ACCESSOR(int, InnerIterations, B2F_BROX_INNER_ITERATIONS)
    B2F_EXT_ACCESSOR(int, OuterIterations, B2F_BROX_OUTER_ITERATIONS)
    B2F_EXT_ACCESSOR(int, SolverIterations, B2F_BROX_SOLVER_ITERATIONS)
    BroxOpticalFlow() {
        b2f_brox_params p{0.197f, 50.0f, 0.8f, 10, 77, 10};
        own(b2f_brox_create(&p, &h_), "createOptFlow_Brox_CUDA");
    }
};

/** cv::superres::PyrLKOpticalFlow (optical_flow.hpp:180-196), createOptFlow_PyrLK_CUDA. */
class PyrLKOpticalFlow : public impl::WrapperBase {
public:
    int getWindowSize() const { return static_cast<int>(get(B2F_LK_WIN_WIDTH)); }
    void setWindowSize(int v) {
        set(B2F_LK_WIN_WIDTH, v);
        set(B2F_LK_WIN_HEIGHT, v);
    }
    B2F_EXT_ACCESSOR(int, MaxLevel, B2F_LK_MAX_LEVEL)
    B2F_EXT_ACCESSOR(int, Iterations, B2F_LK_ITERS)
    PyrLKOpticalFlow() { own(b2f_denselk_create(nullptr, &h_), "createOptFlow_PyrLK_CUDA"); }
};

#undef B2F_EXT_ACCESSOR

inline Ptr<FarnebackOpticalFlow> createOptFlow_Farneback_CUDA() { return detail::make<FarnebackOpticalFlow>(); }
inline Ptr<DualTVL1OpticalFlow> createOptFlow_DualTVL1_CUDA() { return detail::make<DualTVL1OpticalFlow>(); }
inline Ptr<BroxOpticalFlow> createOptFlow_Brox_CUDA() { return detail::make<BroxOpticalFlow>(); }
inline Ptr<PyrLKOpticalFlow> createOptFlow_PyrLK_CUDA() { return detail::make<PyrLKOpticalFlow>(); }

/** cv::superres::SuperResolution as createSuperResolution_BTVL1_CUDA builds it (superres.hpp:87-200): the pull
 *  schedule of btv_l1_cuda.cpp:483-582 runs in the library; nextFrame feeds it frames while it asks for them. */
class SuperResolution : public Algorithm, public FrameSource {
public:
    SuperResolution() {
        flow_ = createOptFlow_Farneback_CUDA();
        const int st = b2f_superres_create(nullptr, flow_->engine(), &h_);
        if (st != B2F_OK) detail::fail(st, "createSuperResolution_BTVL1_CUDA");
    }
    ~SuperResolution() override { b2f_superres_destroy(h_); }

    void setInput(const Ptr<FrameSource> &frameSource) {
        source_ = frameSource;
        restart();
    }
    void nextFrame(OutputArray frame) override {
        int wants = 0;
        for (;;) {
            check(b2f_superres_wants_frame(h_, &wants), "nextFrame");
            if (!wants) break;
            GpuMat f;
            source_->nextFrame(f);
            push(f);
        }
        int rows = 0, cols = 0, got = 0;
        if (b2f_superres_output_size(h_, &rows, &cols) != B2F_OK) rows = cols = 1;  // no frame: the pop reports the end
        auto &out = detail::out_create(frame, rows, cols, type_);
        b2f_image o = impl::image(out);
        check(b2f_superres_pop(h_, &o, &got, stream_), "nextFrame");
        if (!got) out = GpuMat();  // _output.release(): the end of the stream
    }
    void reset() override {
        source_->reset();
        restart();
    }
    virtual void collectGarbage() {
        prev_ = GpuMat();
        check(b2f_superres_collect_garbage(h_), "collectGarbage");
    }
    String getDefaultName() const override { return "SuperResolution.BTVL1_CUDA"; }

#define B2F_SR_ACCESSOR(T, Name, ID)                                   \
    T get##Name() const {                                              \
        double v = 0;                                                  \
        b2f_superres_get_param(h_, ID, &v);                            \
        return static_cast<T>(v);                                      \
    }                                                                  \
    void set##Name(T v) { check(b2f_superres_set_param(h_, ID, static_cast<double>(v)), "set" #Name); }
    B2F_SR_ACCESSOR(int, Scale, B2F_SR_SCALE)
    B2F_SR_ACCESSOR(int, Iterations, B2F_SR_ITERATIONS)
    B2F_SR_ACCESSOR(double, Tau, B2F_SR_TAU)
    B2F_SR_ACCESSOR(double, Lambda, B2F_SR_LAMBDA)
    B2F_SR_ACCESSOR(double, Alpha, B2F_SR_ALPHA)
    B2F_SR_ACCESSOR(int, KernelSize, B2F_SR_BTV_KERNEL_SIZE)
    B2F_SR_ACCESSOR(int, BlurKernelSize, B2F_SR_BLUR_KERNEL_SIZE)
    B2F_SR_ACCESSOR(double, BlurSigma, B2F_SR_BLUR_SIGMA)
    B2F_SR_ACCESSOR(int, TemporalAreaRadius, B2F_SR_TEMPORAL_AREA_RADIUS)
#undef B2F_SR_ACCESSOR

    Ptr<DenseOpticalFlowExt> getOpticalFlow() const { return flow_; }
    void setOpticalFlow(const Ptr<DenseOpticalFlowExt> &val) {
        check(b2f_superres_set_flow(h_, val->engine()), "setOpticalFlow");
        flow_ = val;
    }

private:
    b2f_superres *h_ = nullptr;
    Ptr<FrameSource> source_;
    Ptr<DenseOpticalFlowExt> flow_;
    GpuMat prev_;
    int type_ = B2F_8UC1;
    cudaStream_t stream_ = nullptr;

    void check(int st, const char *where) const {
        if (st != B2F_OK) detail::fail(st, where);
    }
    void restart() {
        prev_ = GpuMat();
        check(b2f_superres_reset(h_), "setInput");
    }
    void push(const GpuMat &f) {
        if (f.empty()) {
            check(flow_->engine() ? b2f_superres_push(h_, nullptr, stream_)
                                  : b2f_superres_push_flows(h_, nullptr, nullptr, nullptr, nullptr, nullptr, stream_),
                  "nextFrame");
            return;
        }
        type_ = f.type();
        b2f_image img = impl::image(f);
        if (flow_->engine()) {
            check(b2f_superres_push(h_, &img, stream_), "nextFrame");
        } else if (prev_.empty()) {
            check(b2f_superres_push_flows(h_, &img, nullptr, nullptr, nullptr, nullptr, stream_), "nextFrame");
        } else {
            // readNextFrame (btv_l1_cuda.cpp:547-548): calc(prev, cur) and calc(cur, prev), planar
            GpuMat fu, fv, bu, bv;
            flow_->calc(prev_, f, fu, fv);
            flow_->calc(f, prev_, bu, bv);
            b2f_image a = impl::image(fu), b = impl::image(fv), c = impl::image(bu), d = impl::image(bv);
            check(b2f_superres_push_flows(h_, &img, &a, &b, &c, &d, stream_), "nextFrame");
        }
        // curFrame_.copyTo(prevFrame_): a deep copy, the source may reuse its buffer
        prev_.create(f.rows, f.cols, f.type());
        check(cudaMemcpy2DAsync(prev_.data, prev_.step, f.data, f.step, (size_t)f.cols * f.elemSize(), f.rows,
                                cudaMemcpyDeviceToDevice, stream_) == cudaSuccess ? B2F_OK : B2F_CUDA_ERROR,
              "nextFrame");
    }
};

inline Ptr<SuperResolution> createSuperResolution_BTVL1_CUDA() { return detail::make<SuperResolution>(); }

}  // namespace superres
}  // namespace b200flow
