// cudaimgproc_compat.hpp -- header-only C++ adapter reproducing the reference's CUDA corner API on top of the C ABI
// (b2f_harris_create, b2f_mineig_create, b2f_corners_compute, b2f_gftt_* in include/b200flow.h).
//
// Reference interface mirrored (modules/cudaimgproc/include/opencv2/cudaimgproc.hpp):
//   CornernessCriteria, createHarrisCorner, createMinEigenValCorner        :538-579
//   CornersDetector, createGoodFeaturesToTrackDetector                     :581-620
// Same class names, method names and argument order, so a call site only changes its namespace:
//   namespace cu = b200flow::cuda;
// detect() writes a 1 x N CV_32FC2 GpuMat (released when N is 0, as the reference does); reading N is its one 4-byte
// host read, where the reference synchronises, downloads every candidate and uploads the result.
#pragma once

#include "cudaoptflow_compat.hpp"

namespace b200flow {
namespace cuda {

enum { BORDER_REPLICATE = 1, BORDER_REFLECT = 2, BORDER_REFLECT101 = 4, BORDER_REFLECT_101 = 4 };

namespace impl {
inline b2f_image corner_image(const GpuMat &m) { return b2f_image{m.data, m.step, m.rows, m.cols, m.type()}; }

class CornersHandle {
public:
    ~CornersHandle() { b2f_corners_destroy(h_); }
    CornersHandle() = default;
    CornersHandle(const CornersHandle &) = delete;
    CornersHandle &operator=(const CornersHandle &) = delete;

protected:
    b2f_corners *h_ = nullptr;
    void check(int st, const char *where) const {
        if (st != B2F_OK) detail::fail(st, where);
    }
};
}  // namespace impl

/** cv::cuda::CornernessCriteria (cudaimgproc.hpp:538-567). */
class CornernessCriteria : public Algorithm, protected impl::CornersHandle {
public:
    CornernessCriteria(bool harris, int srcType, int blockSize, int ksize, double k, int borderType) {
        check(harris ? b2f_harris_create(srcType, blockSize, ksize, k, borderType, &h_)
                     : b2f_mineig_create(srcType, blockSize, ksize, borderType, &h_),
              harris ? "createHarrisCorner" : "createMinEigenValCorner");
    }
    /** compute(src, dst, stream): dst becomes a CV_32FC1 GpuMat of src's size. */
    void compute(InputArray src, OutputArray dst, Stream &stream = Stream::Null()) {
        const auto &s = detail::in_mat(src);
        auto &d = detail::out_create(dst, s.rows, s.cols, B2F_32FC1);
        b2f_image is = impl::corner_image(s), id = impl::corner_image(d);
        check(b2f_corners_compute(h_, &is, &id, detail::raw(stream)), "CornernessCriteria::compute");
    }
};

/** cv::cuda::CornersDetector (cudaimgproc.hpp:581-600): the GoodFeaturesToTrack detector. */
class CornersDetector : public Algorithm, protected impl::CornersHandle {
public:
    CornersDetector(int srcType, int maxCorners, double qualityLevel, double minDistance, int blockSize,
                    bool useHarrisDetector, double harrisK) {
        b2f_gftt_params p{maxCorners, qualityLevel, minDistance, blockSize, useHarrisDetector ? 1 : 0, harrisK};
        check(b2f_gftt_create(srcType, &p, &h_), "createGoodFeaturesToTrackDetector");
    }
    /** detect(image, corners, mask, stream): corners becomes 1 x N CV_32FC2, strongest first. */
    void detect(InputArray image, OutputArray corners, InputArray mask = detail::noArray(),
                Stream &stream = Stream::Null()) {
        const auto &img = detail::in_mat(image);
        const auto &m = detail::in_mat(mask);
        int cap = 0;
        check(b2f_gftt_capacity(h_, img.rows, img.cols, &cap), "CornersDetector::detect");
        buf_.create(1, cap + 1, B2F_32FC2);  // (capacity corners, then the count in the last element)
        float *pts = static_cast<float *>(static_cast<void *>(buf_.data));
        int *count_dev = reinterpret_cast<int *>(pts + 2 * (size_t)cap);
        b2f_image ii = impl::corner_image(img), im = impl::corner_image(m);
        cudaStream_t s = detail::raw(stream);
        check(b2f_gftt_detect(h_, &ii, m.empty() ? nullptr : &im, pts, cap, count_dev, s), "CornersDetector::detect");
        int n = 0;
        check(cudaMemcpyAsync(&n, count_dev, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
                      cudaStreamSynchronize(s) == cudaSuccess ? B2F_OK : B2F_CUDA_ERROR,
              "CornersDetector::detect");
        if (n == 0) {
            release(corners);  // gftt.cpp:126-130
            return;
        }
        auto &out = detail::out_create(corners, 1, n, B2F_32FC2);
        check(cudaMemcpyAsync(out.data, pts, sizeof(float) * 2 * (size_t)n, cudaMemcpyDeviceToDevice, s) == cudaSuccess
                  ? B2F_OK : B2F_CUDA_ERROR,
              "CornersDetector::detect");
    }
    void setMaxCorners(int maxCorners) { update([&](b2f_gftt_params &p) { p.max_corners = maxCorners; }); }
    void setMinDistance(double minDistance) { update([&](b2f_gftt_params &p) { p.min_distance = minDistance; }); }

private:
    GpuMat buf_;
    template <class F> void update(F &&f) {
        b2f_gftt_params p;
        check(b2f_gftt_get_params(h_, &p), "CornersDetector");
        f(p);
        check(b2f_gftt_set_params(h_, &p), "CornersDetector");
    }
#ifdef B200FLOW_WITH_OPENCV
    static void release(OutputArray a) { a.release(); }
#else
    static void release(OutputArray a) { a = GpuMat(); }
#endif
};

/** cv::cuda::createHarrisCorner (cudaimgproc.hpp:569-575). */
inline Ptr<CornernessCriteria> createHarrisCorner(int srcType, int blockSize, int ksize, double k,
                                                  int borderType = BORDER_REFLECT101) {
    return detail::make<CornernessCriteria>(true, srcType, blockSize, ksize, k, borderType);
}

/** cv::cuda::createMinEigenValCorner (cudaimgproc.hpp:577-579). */
inline Ptr<CornernessCriteria> createMinEigenValCorner(int srcType, int blockSize, int ksize,
                                                       int borderType = BORDER_REFLECT101) {
    return detail::make<CornernessCriteria>(false, srcType, blockSize, ksize, 0.0, borderType);
}

/** cv::cuda::createGoodFeaturesToTrackDetector (cudaimgproc.hpp:610-620). */
inline Ptr<CornersDetector> createGoodFeaturesToTrackDetector(int srcType, int maxCorners = 1000,
                                                             double qualityLevel = 0.01, double minDistance = 0.0,
                                                             int blockSize = 3, bool useHarrisDetector = false,
                                                             double harrisK = 0.04) {
    return detail::make<CornersDetector>(srcType, maxCorners, qualityLevel, minDistance, blockSize, useHarrisDetector,
                                         harrisK);
}

}  // namespace cuda
}  // namespace b200flow
