// Exercises the C++ VariationalRefinement adapter (cudaoptflow_compat.hpp) the way a call site polishing a flow does:
// upload two 8-bit frames and an initial CV_32FC2 flow, create() + setters, calc on a stream (the flow refined in place),
// then calcUV on the split planes, download.  Writes the refined flow (rows x cols x 2 float32) and the planar result
// (u plane then v plane); tests/test_varref_gpu.py compares them bit for bit with oracle/dis_model.py.  An empty flow
// must be refused with the adapter's exception.
//   usage: test_varref_compat rows cols i0.raw i1.raw flow.raw out.raw out_uv.raw
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "b200flow/cudaoptflow_compat.hpp"

namespace cu = b200flow::cuda;
using b200flow::shim::CV_8U;
using b200flow::shim::CV_32FC1;
using b200flow::shim::CV_32FC2;

static bool read_file(const char *path, void *dst, size_t n) {
    FILE *f = fopen(path, "rb");
    if (!f) return false;
    const bool ok = fread(dst, 1, n, f) == n;
    fclose(f);
    return ok;
}

int main(int argc, char **argv) {
    if (argc < 8) return 2;
    const int rows = atoi(argv[1]), cols = atoi(argv[2]);
    const size_t n = (size_t)rows * cols;
    std::vector<unsigned char> h0(n), h1(n);
    std::vector<float> hf(2 * n);
    if (!read_file(argv[3], h0.data(), n) || !read_file(argv[4], h1.data(), n) ||
        !read_file(argv[5], hf.data(), 8 * n))
        return 2;
    std::vector<float> hu(n), hv(n);
    for (size_t i = 0; i < n; ++i) {
        hu[i] = hf[2 * i];
        hv[i] = hf[2 * i + 1];
    }
    cudaStream_t cs;
    cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
    cu::Stream stream(cs);
    try {
        cu::GpuMat i0(rows, cols, CV_8U), i1(rows, cols, CV_8U), flow(rows, cols, CV_32FC2);
        cu::GpuMat u(rows, cols, CV_32FC1), v(rows, cols, CV_32FC1);
        i0.upload(h0.data(), cols, stream);
        i1.upload(h1.data(), cols, stream);
        flow.upload(hf.data(), (size_t)cols * 8, stream);
        u.upload(hu.data(), (size_t)cols * 4, stream);
        v.upload(hv.data(), (size_t)cols * 4, stream);
        auto vr = cu::VariationalRefinement::create();
        if (vr->getDefaultName() != "my_object" || vr->getFixedPointIterations() != 5 || vr->getOmega() != 1.6f)
            return 3;
        vr->setSorIterations(7);
        vr->setEpsilon(0.01f);
        vr->calc(i0, i1, flow, stream);
        vr->calcUV(i0, i1, u, v, stream);
        std::vector<float> out(2 * n), ou(n), ov(n);
        flow.download(out.data(), (size_t)cols * 8, stream);
        u.download(ou.data(), (size_t)cols * 4, stream);
        v.download(ov.data(), (size_t)cols * 4, stream);
        stream.waitForCompletion();
        FILE *o = fopen(argv[6], "wb");
        fwrite(out.data(), 4, out.size(), o);
        fclose(o);
        o = fopen(argv[7], "wb");
        fwrite(ou.data(), 4, n, o);
        fwrite(ov.data(), 4, n, o);
        fclose(o);
        // the flow is always read: an empty one is refused, as cv2's calc asserts on it
        bool threw = false;
        try {
            cu::GpuMat none;
            vr->calc(i0, i1, none, stream);
        } catch (const std::exception &) {
            threw = true;
        }
        if (!threw) return 4;
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    cudaStreamDestroy(cs);
    return 0;
}
