// video_compat.hpp -- header-only C++ adapter for the video module's pyramidal Lucas-Kanade tracker on top of the C ABI
// (b2f_lkpyr_* in include/b200flow.h).
//
// Interface mirrored (modules/video/include/opencv2/video/tracking.hpp): buildOpticalFlowPyramid,
// calcOpticalFlowPyrLK, SparsePyrLKOpticalFlow (create, calc, the getters and setters).  These live in namespace
// b200flow, as cv:: holds them next to cv::cuda::, and work on device memory: frames are 8U GpuMats (or an
// OpticalFlowPyramid built from one), points 1 x N CV_32FC2 GpuMats, status 1 x N CV_8UC1 and err 1 x N CV_32FC1.
// Results equal cv::calcOpticalFlowPyrLK bit for bit; b200flow::cuda::SparsePyrLKOpticalFlow is the cv::cuda tracker.
// The video module's Farneback flow (calcOpticalFlowFarneback, FarnebackOpticalFlow; b2f_optflowgf_*) is here too.
#pragma once

#include <map>

#include "cudaoptflow_compat.hpp"

namespace b200flow {

using cuda::GpuMat;
using cuda::Ptr;
using cuda::Size;
using cuda::Stream;

enum { OPTFLOW_LK_GET_MIN_EIGENVALS = 8 };
enum { BORDER_CONSTANT = 0, BORDER_REFLECT_101 = 4 };

/** cv::TermCriteria, as the tracker reads it. */
struct TermCriteria {
    enum { COUNT = 1, MAX_ITER = 1, EPS = 2 };
    int type = COUNT + EPS;
    int maxCount = 30;
    double epsilon = 0.01;
    TermCriteria() = default;
    TermCriteria(int t, int m, double e) : type(t), maxCount(m), epsilon(e) {}
};

/** buildOpticalFlowPyramid's output on the device (cv2's std::vector<Mat>, borders included). */
class OpticalFlowPyramid {
public:
    OpticalFlowPyramid() {
        if (b2f_lkpyr_pyramid_create(&p_) != B2F_OK) detail::fail(B2F_OUT_OF_MEMORY, "OpticalFlowPyramid");
    }
    ~OpticalFlowPyramid() { b2f_lkpyr_pyramid_destroy(p_); }
    OpticalFlowPyramid(const OpticalFlowPyramid &) = delete;
    OpticalFlowPyramid &operator=(const OpticalFlowPyramid &) = delete;
    int levels() const {
        int n = 0;
        b2f_lkpyr_pyramid_info(p_, &n, nullptr, nullptr, nullptr);
        return n;
    }
    /** level `i` (or its derivatives) with its border, as a b2f_image view of the pyramid's memory */
    b2f_image level(int i, bool deriv = false) const {
        b2f_image v{};
        const int st = b2f_lkpyr_pyramid_level(p_, i, deriv ? 1 : 0, &v);
        if (st != B2F_OK) detail::fail(st, "OpticalFlowPyramid::level");
        return v;
    }
    b2f_lkpyr_pyramid *raw() const { return p_; }

private:
    b2f_lkpyr_pyramid *p_ = nullptr;
};

/** A frame argument: an 8U GpuMat or a pyramid. */
struct LkFrame {
    const GpuMat *mat = nullptr;
    const OpticalFlowPyramid *pyr = nullptr;
    LkFrame(const GpuMat &m) : mat(&m) {}                 // NOLINT: implicit, as InputArray is
    LkFrame(const OpticalFlowPyramid &p) : pyr(&p) {}     // NOLINT
};

/** cv::buildOpticalFlowPyramid; returns the last level built. */
inline int buildOpticalFlowPyramid(const GpuMat &img, OpticalFlowPyramid &pyramid, Size winSize, int maxLevel,
                                   bool withDerivatives = true, int pyrBorder = BORDER_REFLECT_101,
                                   int derivBorder = BORDER_CONSTANT, bool /*tryReuseInputImage*/ = true,
                                   Stream &stream = Stream::Null()) {
    b2f_image im{img.data, img.step, img.rows, img.cols, img.type()};
    int out = 0;
    const int st = b2f_lkpyr_build_pyramid(&im, winSize.width, winSize.height, maxLevel, withDerivatives ? 1 : 0, pyrBorder,
                                           derivBorder, pyramid.raw(), &out, detail::raw(stream));
    if (st != B2F_OK) detail::fail(st, "buildOpticalFlowPyramid");
    return out;
}

/** cv::SparsePyrLKOpticalFlow (tracking.hpp). */
class SparsePyrLKOpticalFlow : public cuda::Algorithm {
public:
    SparsePyrLKOpticalFlow(Size winSize, int maxLevel, TermCriteria crit, int flags, double minEigThreshold) {
        b2f_lkpyr_params p{winSize.width, winSize.height, maxLevel, crit.type, crit.maxCount, crit.epsilon, flags,
                           minEigThreshold};
        check(b2f_lkpyr_create(&p, &h_), "SparsePyrLKOpticalFlow::create");
    }
    ~SparsePyrLKOpticalFlow() { b2f_lkpyr_destroy(h_); }
    static Ptr<SparsePyrLKOpticalFlow> create(Size winSize = Size(21, 21), int maxLevel = 3,
                                              TermCriteria crit = TermCriteria(TermCriteria::COUNT + TermCriteria::EPS, 30, 0.01),
                                              int flags = 0, double minEigThreshold = 1e-4) {
        return detail::make<SparsePyrLKOpticalFlow>(winSize, maxLevel, crit, flags, minEigThreshold);
    }

    /** calc(prevImg, nextImg, prevPts, nextPts, status, err, stream): nextPts, status and err are (re)allocated 1 x N
     * unless nextPts is read as the initial estimate (OPTFLOW_USE_INITIAL_FLOW). */
    void calc(LkFrame prevImg, LkFrame nextImg, const GpuMat &prevPts, GpuMat &nextPts, GpuMat &status, GpuMat &err,
              Stream &stream = Stream::Null()) {
        const int n = prevPts.rows * prevPts.cols;
        if (prevPts.type() != B2F_32FC2 || (prevPts.rows != 1 && prevPts.cols != 1)) detail::fail(B2F_BAD_ARG, "calc");
        if (!(params().flags & B2F_LKPYR_USE_INITIAL_FLOW)) nextPts.create(1, n, B2F_32FC2);
        if (nextPts.rows * nextPts.cols != n || nextPts.type() != B2F_32FC2) detail::fail(B2F_SIZE_MISMATCH, "calc");
        status.create(1, n, B2F_8UC1);
        err.create(1, n, B2F_32FC1);
        b2f_image a{}, b{};
        if (prevImg.mat) a = b2f_image{prevImg.mat->data, prevImg.mat->step, prevImg.mat->rows, prevImg.mat->cols, prevImg.mat->type()};
        if (nextImg.mat) b = b2f_image{nextImg.mat->data, nextImg.mat->step, nextImg.mat->rows, nextImg.mat->cols, nextImg.mat->type()};
        check(b2f_lkpyr_calc(h_, prevImg.mat ? &a : nullptr, prevImg.pyr ? prevImg.pyr->raw() : nullptr,
                             nextImg.mat ? &b : nullptr, nextImg.pyr ? nextImg.pyr->raw() : nullptr,
                             static_cast<const float *>(static_cast<const void *>(prevPts.data)),
                             static_cast<float *>(static_cast<void *>(nextPts.data)), static_cast<unsigned char *>(status.data),
                             static_cast<float *>(static_cast<void *>(err.data)), n, detail::raw(stream)),
              "SparsePyrLKOpticalFlow::calc");
    }

    Size getWinSize() const { return Size(params().win_width, params().win_height); }
    void setWinSize(Size s) { update([&](b2f_lkpyr_params &p) { p.win_width = s.width; p.win_height = s.height; }); }
    int getMaxLevel() const { return params().max_level; }
    void setMaxLevel(int v) { update([&](b2f_lkpyr_params &p) { p.max_level = v; }); }
    TermCriteria getTermCriteria() const {
        const b2f_lkpyr_params p = params();
        return TermCriteria(p.criteria_type, p.max_count, p.epsilon);
    }
    void setTermCriteria(const TermCriteria &c) {
        update([&](b2f_lkpyr_params &p) { p.criteria_type = c.type; p.max_count = c.maxCount; p.epsilon = c.epsilon; });
    }
    int getFlags() const { return params().flags; }
    void setFlags(int v) { update([&](b2f_lkpyr_params &p) { p.flags = v; }); }
    double getMinEigThreshold() const { return params().min_eig_threshold; }
    void setMinEigThreshold(double v) { update([&](b2f_lkpyr_params &p) { p.min_eig_threshold = v; }); }
    cuda::String getDefaultName() const { return "SparsePyrLKOpticalFlow"; }

private:
    b2f_lkpyr *h_ = nullptr;
    static void check(int st, const char *where) {
        if (st != B2F_OK) detail::fail(st, where);
    }
    b2f_lkpyr_params params() const {
        b2f_lkpyr_params p{};
        b2f_lkpyr_get_params(h_, &p);
        return p;
    }
    template <class F>
    void update(F &&f) {
        b2f_lkpyr_params p = params();
        f(p);
        check(b2f_lkpyr_set_params(h_, &p), "SparsePyrLKOpticalFlow::set");
    }
};

/** cv::calcOpticalFlowPyrLK. */
inline void calcOpticalFlowPyrLK(LkFrame prevImg, LkFrame nextImg, const GpuMat &prevPts, GpuMat &nextPts, GpuMat &status,
                                 GpuMat &err, Size winSize = Size(21, 21), int maxLevel = 3,
                                 TermCriteria criteria = TermCriteria(TermCriteria::COUNT + TermCriteria::EPS, 30, 0.01),
                                 int flags = 0, double minEigThreshold = 1e-4, Stream &stream = Stream::Null()) {
    SparsePyrLKOpticalFlow lk(winSize, maxLevel, criteria, flags, minEigThreshold);
    lk.calc(prevImg, nextImg, prevPts, nextPts, status, err, stream);
}

/** cv::FarnebackOpticalFlow (the video module's class; b2f_optflowgf_create): results equal cv2's portable CPU path bit
 * for bit.  b200flow::cuda::FarnebackOpticalFlow is the cv::cuda class. */
#define B2F_GF_ACCESSOR(T, Name, ID)                        \
    T get##Name() const { return static_cast<T>(get(ID)); } \
    void set##Name(T v) { set(ID, static_cast<double>(v)); }

class FarnebackOpticalFlow : public cuda::DenseOpticalFlow, protected cuda::impl::HandleOwner {
public:
    B2F_GF_ACCESSOR(int, NumLevels, B2F_FARN_NUM_LEVELS)
    B2F_GF_ACCESSOR(double, PyrScale, B2F_FARN_PYR_SCALE)
    B2F_GF_ACCESSOR(bool, FastPyramids, B2F_FARN_FAST_PYRAMIDS)
    B2F_GF_ACCESSOR(int, WinSize, B2F_FARN_WIN_SIZE)
    B2F_GF_ACCESSOR(int, NumIters, B2F_FARN_NUM_ITERS)
    B2F_GF_ACCESSOR(int, PolyN, B2F_FARN_POLY_N)
    B2F_GF_ACCESSOR(double, PolySigma, B2F_FARN_POLY_SIGMA)
    B2F_GF_ACCESSOR(int, Flags, B2F_FARN_FLAGS)

    void calc(cuda::InputArray I0, cuda::InputArray I1, cuda::InputOutputArray flow,
              Stream &stream = Stream::Null()) override {
        run(I0, I1, flow, stream, (getFlags() & cuda::OPTFLOW_USE_INITIAL_FLOW) != 0);
    }
    cuda::String getDefaultName() const override { return b2f_default_name(h_); }

    static Ptr<FarnebackOpticalFlow> create(int numLevels = 5, double pyrScale = 0.5, bool fastPyramids = false,
                                            int winSize = 13, int numIters = 10, int polyN = 5,
                                            double polySigma = 1.1, int flags = 0) {
        b2f_farneback_params p{numLevels, pyrScale, fastPyramids, winSize, numIters, polyN, polySigma, flags};
        auto o = detail::make<FarnebackOpticalFlow>();
        const int st = b2f_optflowgf_create(&p, &o->h_);
        if (st != B2F_OK) detail::fail(st, "FarnebackOpticalFlow::create");
        return o;
    }
};

#undef B2F_GF_ACCESSOR

/** cv::calcOpticalFlowFarneback, on one handle per host thread and device whose workspace persists between calls.
 * Calls on different streams are safe: the handle orders a call on another stream after the previous call. */
inline void calcOpticalFlowFarneback(const GpuMat &prev, const GpuMat &next, GpuMat &flow, double pyr_scale, int levels,
                                     int winsize, int iterations, int poly_n, double poly_sigma, int flags,
                                     Stream &stream = Stream::Null()) {
    // a handle belongs to the device of its first call
    thread_local std::map<int, Ptr<FarnebackOpticalFlow>> handles;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) detail::fail(B2F_NO_DEVICE, "calcOpticalFlowFarneback");
    Ptr<FarnebackOpticalFlow> &fb = handles[dev];
    if (!fb) fb = FarnebackOpticalFlow::create();
    fb->setPyrScale(pyr_scale);
    fb->setNumLevels(levels);
    fb->setWinSize(winsize);
    fb->setNumIters(iterations);
    fb->setPolyN(poly_n);
    fb->setPolySigma(poly_sigma);
    fb->setFlags(flags);
    fb->calc(prev, next, flow, stream);
}

}  // namespace b200flow
