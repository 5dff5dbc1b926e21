// Exercises the C++ corner adapter (cudaimgproc_compat.hpp) the way a cudaimgproc call site does
// (cf. modules/cudaimgproc/test/test_corners.cpp, test_gftt.cpp): upload an 8-bit image, createHarrisCorner(...)->compute,
// createGoodFeaturesToTrackDetector(...)->detect on a stream, download.  Writes the response (float32, rows x cols) and
// the corners (int32 N, then N (x, y) float32 pairs); tests/test_cudaimgproc_compat_gpu.py compares them bit for bit
// with oracle/corners_model.py.  A flat image must give an empty (released) corner matrix.
//   usage: test_cudaimgproc_compat rows cols in.raw eig.raw corners.raw
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "b200flow/cudaimgproc_compat.hpp"

namespace cu = b200flow::cuda;
using b200flow::shim::CV_8U;
using b200flow::shim::CV_32FC2;

int main(int argc, char **argv) {
    if (argc < 6) return 2;
    const int rows = atoi(argv[1]), cols = atoi(argv[2]);
    std::vector<unsigned char> h((size_t)rows * cols);
    FILE *f = fopen(argv[3], "rb");
    if (!f || fread(h.data(), 1, h.size(), f) != h.size()) return 2;
    fclose(f);
    cudaStream_t cs;
    cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
    cu::Stream stream(cs);
    try {
        cu::GpuMat img(rows, cols, CV_8U), eig, corners;
        img.upload(h.data(), cols, stream);
        auto harris = cu::createHarrisCorner(CV_8U, 5, 5, 0.04, cu::BORDER_REFLECT);
        harris->compute(img, eig, stream);
        auto det = cu::createGoodFeaturesToTrackDetector(CV_8U, 1000, 0.01, 0.0);
        det->setMinDistance(3.0);
        det->setMaxCorners(500);
        det->detect(img, corners, cu::GpuMat(), stream);
        std::vector<float> he((size_t)rows * cols), hc(2 * (size_t)corners.cols);
        eig.download(he.data(), (size_t)cols * 4, stream);
        if (!corners.empty()) corners.download(hc.data(), (size_t)corners.cols * 8, stream);
        stream.waitForCompletion();
        if (corners.rows != 1 || corners.type() != CV_32FC2) return 3;
        FILE *o = fopen(argv[4], "wb");
        fwrite(he.data(), 4, he.size(), o);
        fclose(o);
        o = fopen(argv[5], "wb");
        const int n = corners.cols;
        fwrite(&n, 4, 1, o);
        fwrite(hc.data(), 4, hc.size(), o);
        fclose(o);
        // a flat image has no candidate: the output is released, as the reference's detect does
        cu::GpuMat flat(rows, cols, CV_8U);
        cudaMemsetAsync(flat.data, 7, flat.step * rows, cs);
        det->detect(flat, corners, cu::GpuMat(), stream);
        if (!corners.empty()) return 4;
        // a refused argument surfaces as the adapter's exception
        bool threw = false;
        try {
            cu::createGoodFeaturesToTrackDetector(CV_8U, 1000, 0.0);
        } catch (const std::exception &) {
            threw = true;
        }
        if (!threw) return 5;
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    cudaStreamDestroy(cs);
    return 0;
}
