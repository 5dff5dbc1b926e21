// gpumat_shim.hpp -- minimal stand-ins for the OpenCV core types that cross the cudaoptflow API
// (cv::cuda::GpuMat, cv::cuda::Stream, cv::Ptr, cv::Size, cv::Algorithm), used ONLY when the real
// OpenCV headers are not on the include path (they are not in the build container: opencv core is
// external to opencv_contrib).  Field names and meanings follow opencv core's cuda.hpp so that
// cudaoptflow_compat.hpp compiles unchanged against either.
#pragma once
#include <cuda_runtime.h>
#include <memory>
#include <stdexcept>
#include <string>

namespace b200flow {
namespace shim {

enum { CV_8U = 0, CV_32F = 5 };
enum { CV_8UC1 = 0, CV_32FC1 = 5, CV_32FC2 = 13, CV_8UC3 = 16, CV_32FC3 = 21, CV_8UC4 = 24, CV_32FC4 = 29 };

struct Size {
    int width = 0, height = 0;
    Size() = default;
    Size(int w, int h) : width(w), height(h) {}
    bool operator==(const Size &o) const { return width == o.width && height == o.height; }
};

class Exception : public std::runtime_error {
public:
    int code;
    Exception(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

template <class T> using Ptr = std::shared_ptr<T>;
template <class T, class... A> Ptr<T> makePtr(A &&...a) { return std::make_shared<T>(std::forward<A>(a)...); }
using String = std::string;

class Stream {
public:
    Stream() : s_(nullptr) {}
    explicit Stream(cudaStream_t s) : s_(s) {}
    static Stream &Null() {
        static Stream n;
        return n;
    }
    cudaStream_t cudaPtr() const { return s_; }
    void waitForCompletion() const { cudaStreamSynchronize(s_); }

private:
    cudaStream_t s_;
};

// Pitched, reference-counted device matrix: (rows, cols, step [bytes], data, type flag).
class GpuMat {
public:
    int flags = 0, rows = 0, cols = 0;
    size_t step = 0;
    unsigned char *data = nullptr;

    GpuMat() = default;
    GpuMat(int r, int c, int t) { create(r, c, t); }
    // 8U or 32F with 1 to 4 channels (OpenCV's CV_MAKETYPE layout: depth in bits 0-2, channels - 1 above)
    static size_t elemSize(int t) {
        const int d = t & 7;
        return d == CV_8U ? (size_t)((t >> 3) + 1) : d == CV_32F ? (size_t)4 * ((t >> 3) + 1) : 0;
    }
    int type() const { return flags; }
    int channels() const { return (flags >> 3) + 1; }
    int depth() const { return flags & 7; }
    size_t elemSize() const { return elemSize(flags); }
    Size size() const { return Size(cols, rows); }
    bool empty() const { return data == nullptr; }
    void create(int r, int c, int t) {
        if (data && r == rows && c == cols && t == flags) return;
        void *p = nullptr;
        size_t pitch = 0;
        if (cudaMallocPitch(&p, &pitch, (size_t)c * elemSize(t), r) != cudaSuccess)
            throw Exception(-217, "cudaMallocPitch failed");  // GpuApiCallError
        hold_ = std::shared_ptr<void>(p, [](void *q) { cudaFree(q); });
        data = static_cast<unsigned char *>(p);
        step = pitch;
        rows = r;
        cols = c;
        flags = t;
    }
    void create(Size s, int t) { create(s.height, s.width, t); }
    void upload(const void *host, size_t host_step, Stream &s = Stream::Null()) {
        cudaMemcpy2DAsync(data, step, host, host_step, (size_t)cols * elemSize(), rows, cudaMemcpyHostToDevice, s.cudaPtr());
    }
    void download(void *host, size_t host_step, Stream &s = Stream::Null()) const {
        cudaMemcpy2DAsync(host, host_step, data, step, (size_t)cols * elemSize(), rows, cudaMemcpyDeviceToHost, s.cudaPtr());
    }

private:
    std::shared_ptr<void> hold_;
};

class Algorithm {
public:
    virtual ~Algorithm() {}
    virtual String getDefaultName() const { return "my_object"; }
};

typedef const GpuMat &InputArray;
typedef GpuMat &InputOutputArray;
typedef GpuMat &OutputArray;
// cv::noArray(): the "not wanted" output; recognised by address
inline GpuMat &noArray() {
    static GpuMat none;
    return none;
}

}  // namespace shim
}  // namespace b200flow
