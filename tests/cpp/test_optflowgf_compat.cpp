// Exercises the C++ adapter of the video module's Farneback flow (video_compat.hpp) the way a caller of
// cv::calcOpticalFlowFarneback does: two 64 x 80 8-bit frame pairs, each run through b200flow::calcOpticalFlowFarneback
// on its own non-blocking stream, back to back with no synchronisation in between (the free function's one handle per
// thread must order the second call after the first); then the first pair again through a FarnebackOpticalFlow made
// with create() and its setters, which must agree with the free function.  Prints both flows (64 x 80 x 2 float32) as
// one hex string each; tests/test_optflowgf_gpu.py compares them with cv2.
#include <cstdio>
#include <cstring>
#include <vector>

#include "b200flow/video_compat.hpp"

using b200flow::shim::CV_8U;

static void frame(std::vector<unsigned char> &h, int rows, int cols, int k) {
    h.resize((size_t)rows * cols);
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) h[(size_t)y * cols + x] = (unsigned char)(((x * 7 + y * 3 + k * 5) % 64) * 4);
}

static void print_hex(const std::vector<float> &a) {
    const unsigned char *p = reinterpret_cast<const unsigned char *>(a.data());
    for (size_t i = 0; i < a.size() * 4; ++i) printf("%02x", p[i]);
    printf("\n");
}

int main() {
    const int rows = 64, cols = 80;
    std::vector<unsigned char> h[3];
    for (int k = 0; k < 3; ++k) frame(h[k], rows, cols, k);
    cudaStream_t sa, sb;
    cudaStreamCreateWithFlags(&sa, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&sb, cudaStreamNonBlocking);
    b200flow::Stream A(sa), B(sb);
    std::vector<float> a((size_t)rows * cols * 2), b(a.size()), c(a.size());
    try {
        b200flow::GpuMat f0(rows, cols, CV_8U), f1(rows, cols, CV_8U), f2(rows, cols, CV_8U), flowA, flowB, flowC;
        f0.upload(h[0].data(), cols, A);
        f1.upload(h[1].data(), cols, A);
        f2.upload(h[2].data(), cols, A);
        A.waitForCompletion();
        // pair (0, 1) on A, then pair (0, 2) on B at once: B's call may not overwrite A's workspace early
        b200flow::calcOpticalFlowFarneback(f0, f1, flowA, 0.5, 3, 9, 3, 5, 1.1, 0, A);
        b200flow::calcOpticalFlowFarneback(f0, f2, flowB, 0.5, 3, 9, 3, 5, 1.1, 0, B);
        flowA.download(a.data(), (size_t)cols * 8, A);
        flowB.download(b.data(), (size_t)cols * 8, B);
        auto fb = b200flow::FarnebackOpticalFlow::create();
        fb->setNumLevels(3);
        fb->setWinSize(9);
        fb->setNumIters(3);
        if (fb->getDefaultName() != "DenseOpticalFlow.FarnebackOpticalFlow") return 3;
        fb->calc(f0, f1, flowC, B);
        flowC.download(c.data(), (size_t)cols * 8, B);
        A.waitForCompletion();
        B.waitForCompletion();
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    cudaStreamDestroy(sa);
    cudaStreamDestroy(sb);
    if (memcmp(a.data(), c.data(), a.size() * 4) != 0) return 4;
    print_hex(a);
    print_hex(b);
    return 0;
}
