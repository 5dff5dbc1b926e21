// Exercises the C++ adapter of the video module's tracker (video_compat.hpp) the way a KLT loop does: upload two 8-bit
// frames and a 1 x N CV_32FC2 point list, track them with b200flow::calcOpticalFlowPyrLK, then three times with one
// SparsePyrLKOpticalFlow on pyramids created and destroyed in each loop iteration, on a stream.  Writes every result
// (N (x, y) float32 pairs, N status bytes, N float32 errors, four times); tests/test_lkpyramid_gpu.py compares them with oracle/lkpyramid_model.py.
//   usage: test_lkpyramid_compat rows cols n in0.raw in1.raw pts.raw out.raw
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "b200flow/video_compat.hpp"

using b200flow::shim::CV_32FC2;
using b200flow::shim::CV_8U;

static bool read_all(const char *path, void *dst, size_t n) {
    FILE *f = fopen(path, "rb");
    const bool ok = f && fread(dst, 1, n, f) == n;
    if (f) fclose(f);
    return ok;
}

int main(int argc, char **argv) {
    if (argc < 8) return 2;
    const int rows = atoi(argv[1]), cols = atoi(argv[2]), n = atoi(argv[3]);
    std::vector<unsigned char> h0((size_t)rows * cols), h1(h0.size());
    std::vector<float> hp(2 * (size_t)n);
    if (!read_all(argv[4], h0.data(), h0.size()) || !read_all(argv[5], h1.data(), h1.size()) ||
        !read_all(argv[6], hp.data(), hp.size() * 4))
        return 2;
    cudaStream_t cs;
    cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
    b200flow::Stream stream(cs);
    std::vector<unsigned char> out;
    try {
        b200flow::GpuMat f0(rows, cols, CV_8U), f1(rows, cols, CV_8U), pts(1, n, CV_32FC2), nxt, st, err;
        f0.upload(h0.data(), cols, stream);
        f1.upload(h1.data(), cols, stream);
        pts.upload(hp.data(), (size_t)n * 8, stream);
        auto dump = [&]() {
            std::vector<unsigned char> buf((size_t)n * 13);
            nxt.download(buf.data(), (size_t)n * 8, stream);
            st.download(buf.data() + (size_t)n * 8, n, stream);
            err.download(buf.data() + (size_t)n * 9, (size_t)n * 4, stream);
            stream.waitForCompletion();
            out.insert(out.end(), buf.begin(), buf.end());
        };
        b200flow::calcOpticalFlowPyrLK(f0, f1, pts, nxt, st, err, b200flow::Size(15, 15), 3,
                                       b200flow::TermCriteria(b200flow::TermCriteria::COUNT + b200flow::TermCriteria::EPS, 30, 0.01),
                                       0, 1e-4, stream);
        dump();
        auto lk = b200flow::SparsePyrLKOpticalFlow::create(b200flow::Size(15, 15), 3);
        lk->setMinEigThreshold(1e-4);
        if (lk->getWinSize().width != 15 || lk->getMaxLevel() != 3 || lk->getTermCriteria().maxCount != 30) return 4;
        // a KLT loop that scopes its pyramids in the loop body: each iteration frees both and builds new ones (of
        // alternating border widths, so the new arenas need not land where the old ones were) on one handle
        for (int it = 0; it < 3; ++it) {
            const int border = it % 2 ? 23 : 15;
            b200flow::OpticalFlowPyramid p0, p1;
            if (b200flow::buildOpticalFlowPyramid(f0, p0, b200flow::Size(border, border), 3, it != 1,
                                                  b200flow::BORDER_REFLECT_101, b200flow::BORDER_CONSTANT, true,
                                                  stream) != p0.levels() - 1)
                return 3;
            b200flow::buildOpticalFlowPyramid(f1, p1, b200flow::Size(border, border), 3, false, b200flow::BORDER_REFLECT_101,
                                              b200flow::BORDER_CONSTANT, true, stream);
            lk->calc(p0, p1, pts, nxt, st, err, stream);
            dump();
        }
        // a border mode the port does not build surfaces as the adapter's exception
        bool threw = false;
        try {
            b200flow::OpticalFlowPyramid bad;
            b200flow::buildOpticalFlowPyramid(f0, bad, b200flow::Size(15, 15), 3, true, 1);
        } catch (const std::exception &) {
            threw = true;
        }
        if (!threw) return 5;
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    FILE *o = fopen(argv[7], "wb");
    fwrite(out.data(), 1, out.size(), o);
    fclose(o);
    cudaStreamDestroy(cs);
    return 0;
}
