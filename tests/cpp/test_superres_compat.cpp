// Exercises the C++ super-resolution adapter (superres_compat.hpp) the way a superres call site does
// (cf. modules/superres/perf/perf_superres.cpp:90-152, samples/super_resolution.cpp): a FrameSource of uploaded frames,
// createSuperResolution_BTVL1_CUDA, the setters, setOpticalFlow, then nextFrame until it returns an empty frame.  Writes
// every 8-bit output; tests/test_superres_compat_gpu.py compares them bit for bit with the Python path.
//   usage: test_superres_compat <zero|farneback|brox> rows cols channels nframes in.raw out.raw
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "b200flow/superres_compat.hpp"

namespace sr = b200flow::superres;

// the reference perf test's ZeroOpticalFlow (perf_superres.cpp:90-115)
class ZeroOpticalFlow : public sr::DenseOpticalFlowExt {
public:
    void calc(sr::InputArray frame0, sr::InputArray, sr::OutputArray flow1, sr::OutputArray flow2) override {
        for (sr::GpuMat *f : {&flow1, &flow2}) {
            f->create(frame0.rows, frame0.cols, 5 /*CV_32FC1*/);
            cudaMemset2D(f->data, f->step, 0, (size_t)frame0.cols * 4, frame0.rows);
        }
    }
    void collectGarbage() override {}
};

class ListSource : public sr::FrameSource {
public:
    std::vector<std::vector<unsigned char>> frames;
    int rows = 0, cols = 0, type = 0, i = 0;
    void nextFrame(sr::OutputArray frame) override {
        if (i >= (int)frames.size()) {
            frame = sr::GpuMat();
            return;
        }
        frame.create(rows, cols, type);
        frame.upload(frames[i++].data(), (size_t)cols * frame.elemSize());
        cudaDeviceSynchronize();
    }
    void reset() override { i = 0; }
};

int main(int argc, char **argv) {
    if (argc < 8) return 2;
    const int rows = atoi(argv[2]), cols = atoi(argv[3]), cn = atoi(argv[4]), n = atoi(argv[5]);
    const size_t fb = (size_t)rows * cols * cn;
    auto src = std::make_shared<ListSource>();
    src->rows = rows, src->cols = cols, src->type = (cn - 1) << 3;
    FILE *f = fopen(argv[6], "rb");
    if (!f) return 2;
    for (int k = 0; k < n; ++k) {
        src->frames.emplace_back(fb);
        if (fread(src->frames.back().data(), 1, fb, f) != fb) return 2;
    }
    fclose(f);
    FILE *out = fopen(argv[7], "wb");
    if (!out) return 2;
    try {
        auto s = sr::createSuperResolution_BTVL1_CUDA();
        if (s->getScale() != 4 || s->getIterations() != 180 || s->getTemporalAreaRadius() != 4 || s->getKernelSize() != 7)
            return 3;
        s->setScale(2);
        s->setIterations(5);
        s->setTemporalAreaRadius(1);
        s->setLambda(0.05);
        if (!strcmp(argv[1], "zero")) {
            s->setOpticalFlow(std::make_shared<ZeroOpticalFlow>());
        } else if (!strcmp(argv[1], "brox")) {
            auto b = sr::createOptFlow_Brox_CUDA();
            b->setOuterIterations(4);
            s->setOpticalFlow(b);
        } else if (strcmp(argv[1], "farneback")) {
            return 2;
        }
        s->setInput(src);
        int produced = 0;
        for (;;) {
            sr::GpuMat frame;
            s->nextFrame(frame);
            if (frame.empty()) break;
            std::vector<unsigned char> h((size_t)frame.rows * frame.cols * frame.elemSize());
            frame.download(h.data(), (size_t)frame.cols * frame.elemSize());
            cudaDeviceSynchronize();
            fwrite(h.data(), 1, h.size(), out);
            ++produced;
        }
        if (produced != n) return 4;
        // refused: an even blur size (cudafilters' odd-size assertion) surfaces as an exception
        s->setBlurKernelSize(4);
        s->setInput(src);
        sr::GpuMat frame;
        try {
            s->nextFrame(frame);
            return 5;
        } catch (const std::exception &) {
        }
    } catch (const std::exception &e) {
        fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    fclose(out);
    return 0;
}
