// video.cu -- video front end (SURVEY.md 8f rank 1): flow between consecutive frames of one stream.
//
// What the reference leaves to the caller (samples/optical_flow.cpp:170-238 uploads both frames of every
// pair and blocks on each calc; test_optflow.cpp:328-334 chains the initial flow by hand) is done here once:
//   * every frame crosses PCIe once -- frame k stays resident as I0 of pair k;
//   * three streams: upload of frame k+1 | solve of pair k | download of flow k-1, joined by events only;
//     push() never synchronises with the device unless `depth` pairs are already in flight;
//   * host frames are staged through an internal pinned ring, so pageable caller memory still gets
//     asynchronous copies and can be reused as soon as push() returns;
//   * optional warm start: pair k starts from flow k-1 (tvl1flow.cpp:203-207,249-256;
//     farneback.cpp:179-188,398-404).
#include <cstring>
#include <vector>

#include "common.cuh"

struct b2f_video {
    b2f_handle *h = nullptr;
    int rows = 0, cols = 0, type = 0, depth = 0;
    bool warm = false;
    int warm_param = 0;        // parameter id that toggles the initial-flow path
    double warm_on = 0, warm_off = 0;
    size_t esz = 0, in_pitch = 0, fl_pitch = 0;
    int nf = 0;                // frame slots
    int64_t pushed = 0;        // frames pushed so far
    cudaStream_t s_copy = nullptr, s_comp = nullptr, s_down = nullptr;
    char *d_frames = nullptr;  // nf * in_pitch * rows
    char *d_flows = nullptr;   // depth * fl_pitch * rows
    char *h_frames = nullptr;  // pinned, nf slots, tightly packed rows
    char *h_flows = nullptr;   // pinned, depth slots, tightly packed rows
    std::vector<cudaEvent_t> copy_done, comp_done, down_done;
    std::vector<int64_t> flow_pair;  // which pair each flow slot currently holds (-1 = none)
    int last_error = 0;
    int device = 0;            // the front end lives on the device that was current at creation

    char *d_frame(int64_t k) const { return d_frames + (size_t)(k % nf) * in_pitch * rows; }
    char *h_frame(int64_t k) const { return h_frames + (size_t)(k % nf) * esz * cols * rows; }
    char *d_flow(int64_t p) const { return d_flows + (size_t)(p % depth) * fl_pitch * rows; }
    char *h_flow(int64_t p) const { return h_flows + (size_t)(p % depth) * 8 * (size_t)cols * rows; }
};

namespace {

int fail(b2f_video *v, cudaError_t e) {
    v->last_error = static_cast<int>(e);
    cudaGetLastError();
    return e == cudaErrorMemoryAllocation ? B2F_OUT_OF_MEMORY : B2F_CUDA_ERROR;
}

#define VCHECK(expr)                                  \
    do {                                              \
        cudaError_t e__ = (expr);                     \
        if (e__ != cudaSuccess) return fail(v, e__);  \
    } while (0)

}  // namespace

extern "C" {

void b2f_video_destroy(b2f_video *v) {
    if (!v) return;
    b2f::DeviceScope dev(v->device);
    if (v->s_copy) cudaStreamSynchronize(v->s_copy);
    if (v->s_comp) cudaStreamSynchronize(v->s_comp);
    if (v->s_down) cudaStreamSynchronize(v->s_down);
    for (auto &e : v->copy_done) cudaEventDestroy(e);
    for (auto &e : v->comp_done) cudaEventDestroy(e);
    for (auto &e : v->down_done) cudaEventDestroy(e);
    if (v->d_frames) cudaFree(v->d_frames);
    if (v->d_flows) cudaFree(v->d_flows);
    if (v->h_frames) cudaFreeHost(v->h_frames);
    if (v->h_flows) cudaFreeHost(v->h_flows);
    if (v->s_copy) cudaStreamDestroy(v->s_copy);
    if (v->s_comp) cudaStreamDestroy(v->s_comp);
    if (v->s_down) cudaStreamDestroy(v->s_down);
    if (v->warm && v->h) b2f_set_param(v->h, v->warm_param, v->warm_off);
    delete v;
}

int b2f_video_create(b2f_handle *h, int rows, int cols, int type, int depth, int warm_start, b2f_video **out) {
    if (!h || !out || rows <= 0 || cols <= 0 || depth < 1 || depth > 64) return B2F_BAD_ARG;
    if (type != B2F_8UC1 && type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
    // VariationalRefinement refines the caller's flow: the frame loop has none, and it reuses its flow slots
    if (h->algo == b2f::ALGO_VARREF) return B2F_BAD_ARG;
    *out = nullptr;
    b2f_video *v = new b2f_video;
    v->h = h;
    cudaGetDevice(&v->device);
    v->rows = rows;
    v->cols = cols;
    v->type = type;
    v->depth = depth;
    v->warm = warm_start != 0;
    if (v->warm) {
        if (h->algo == b2f::ALGO_TVL1) {
            v->warm_param = B2F_TVL1_USE_INITIAL_FLOW;
            v->warm_on = 1;
            v->warm_off = 0;
        } else if (h->algo == b2f::ALGO_FARNEBACK || h->algo == b2f::ALGO_OPTFLOWGF) {
            double flags = 0;
            b2f_get_param(h, B2F_FARN_FLAGS, &flags);
            v->warm_param = B2F_FARN_FLAGS;
            v->warm_off = static_cast<double>(static_cast<int>(flags) & ~B2F_OPTFLOW_USE_INITIAL_FLOW);
            v->warm_on = static_cast<double>(static_cast<int>(flags) | B2F_OPTFLOW_USE_INITIAL_FLOW);
        } else if (h->algo == b2f::ALGO_DIS) {
            v->warm_param = B2F_DIS_USE_INITIAL_FLOW;
            v->warm_on = 1;
            v->warm_off = 0;
        } else {  // Brox, DensePyrLK, DeepFlow and FastBM have no initial-flow path (brox.cpp:129-188, pyrlk.cpp:238-299,
                  // deepflow.cpp:132,146, cudalegacy bm_fast.cpp:62-88)
            delete v;
            return B2F_BAD_ARG;
        }
    }
    v->esz = type == B2F_8UC1 ? 1 : 4;
    v->in_pitch = (cols * v->esz + 255) & ~size_t(255);
    v->fl_pitch = ((size_t)cols * 8 + 255) & ~size_t(255);
    v->nf = depth + 2;
    auto bail = [&](cudaError_t e) {
        const int st = fail(v, e);
        v->warm = false;
        b2f_video_destroy(v);
        return st;
    };
    cudaError_t e;
    if ((e = cudaStreamCreateWithFlags(&v->s_copy, cudaStreamNonBlocking)) != cudaSuccess) return bail(e);
    if ((e = cudaStreamCreateWithFlags(&v->s_comp, cudaStreamNonBlocking)) != cudaSuccess) return bail(e);
    if ((e = cudaStreamCreateWithFlags(&v->s_down, cudaStreamNonBlocking)) != cudaSuccess) return bail(e);
    if ((e = cudaMalloc(&v->d_frames, (size_t)v->nf * v->in_pitch * rows)) != cudaSuccess) return bail(e);
    if ((e = cudaMalloc(&v->d_flows, (size_t)depth * v->fl_pitch * rows)) != cudaSuccess) return bail(e);
    if ((e = cudaMallocHost(&v->h_frames, (size_t)v->nf * v->esz * cols * rows)) != cudaSuccess) return bail(e);
    if ((e = cudaMallocHost(&v->h_flows, (size_t)depth * 8 * cols * rows)) != cudaSuccess) return bail(e);
    if ((e = cudaMemset(v->d_flows, 0, (size_t)depth * v->fl_pitch * rows)) != cudaSuccess) return bail(e);
    auto make_events = [&](std::vector<cudaEvent_t> &ev, int n) {
        ev.resize(n, nullptr);
        for (auto &x : ev)
            if ((e = cudaEventCreateWithFlags(&x, cudaEventDisableTiming)) != cudaSuccess) return false;
        return true;
    };
    if (!make_events(v->copy_done, v->nf) || !make_events(v->comp_done, depth) || !make_events(v->down_done, depth))
        return bail(e);
    v->flow_pair.assign(depth, -1);
    *out = v;
    return B2F_OK;
}

int b2f_video_push(b2f_video *v, const void *host_frame, size_t step, int64_t *pair_index) {
    if (!v || !host_frame) return B2F_BAD_ARG;
    if (step < v->esz * (size_t)v->cols) return B2F_BAD_ARG;
    b2f::DeviceScope dev(v->device);
    const int64_t k = v->pushed;
    const int64_t p = k - 1;  // pair this frame completes
    if (pair_index) *pair_index = p;

    // Flow slot p % depth still holds pair p - depth: its download must have finished (the only host wait).
    // Once it has, every pair <= p - depth is complete, so frame slot k % nf (last read by pair k - nf + ... )
    // and its pinned staging slot are free as well.
    if (p >= v->depth) VCHECK(cudaEventSynchronize(v->down_done[p % v->depth]));
    else if (k >= v->nf) VCHECK(cudaEventSynchronize(v->copy_done[k % v->nf]));

    // stage + upload
    char *hs = v->h_frame(k);
    const size_t row_bytes = v->esz * (size_t)v->cols;
    for (int y = 0; y < v->rows; ++y)
        std::memcpy(hs + (size_t)y * row_bytes, static_cast<const char *>(host_frame) + (size_t)y * step, row_bytes);
    VCHECK(cudaMemcpy2DAsync(v->d_frame(k), v->in_pitch, hs, row_bytes, row_bytes, v->rows, cudaMemcpyHostToDevice,
                             v->s_copy));
    VCHECK(cudaEventRecord(v->copy_done[k % v->nf], v->s_copy));
    v->pushed = k + 1;
    if (p < 0) return B2F_OK;

    // solve pair p on the compute stream once frame k has landed (frame k-1 was waited for by pair p-1 or here)
    VCHECK(cudaStreamWaitEvent(v->s_comp, v->copy_done[k % v->nf], 0));
    if (p == 0) VCHECK(cudaStreamWaitEvent(v->s_comp, v->copy_done[(k - 1) % v->nf], 0));
    if (v->warm) {
        const int st = b2f_set_param(v->h, v->warm_param, p > 0 ? v->warm_on : v->warm_off);
        if (st != B2F_OK) return st;
        if (p > 0 && v->depth > 1)
            VCHECK(cudaMemcpyAsync(v->d_flow(p), v->d_flow(p - 1), v->fl_pitch * v->rows, cudaMemcpyDeviceToDevice,
                                   v->s_comp));
        // depth == 1: the single flow slot already holds flow p-1 and is used in place
    }
    b2f_image I0{v->d_frame(k - 1), v->in_pitch, v->rows, v->cols, v->type};
    b2f_image I1{v->d_frame(k), v->in_pitch, v->rows, v->cols, v->type};
    b2f_image fl{v->d_flow(p), v->fl_pitch, v->rows, v->cols, B2F_32FC2};
    const int st = b2f_calc(v->h, &I0, &I1, &fl, v->s_comp);
    if (st != B2F_OK) return st;
    VCHECK(cudaEventRecord(v->comp_done[p % v->depth], v->s_comp));

    // download flow p
    VCHECK(cudaStreamWaitEvent(v->s_down, v->comp_done[p % v->depth], 0));
    VCHECK(cudaMemcpy2DAsync(v->h_flow(p), 8 * (size_t)v->cols, v->d_flow(p), v->fl_pitch, 8 * (size_t)v->cols, v->rows,
                             cudaMemcpyDeviceToHost, v->s_down));
    VCHECK(cudaEventRecord(v->down_done[p % v->depth], v->s_down));
    // with warm start and depth == 1 the next solve overwrites this slot in place: order it after the download
    if (v->warm && v->depth == 1) VCHECK(cudaStreamWaitEvent(v->s_comp, v->down_done[0], 0));
    v->flow_pair[p % v->depth] = p;
    return B2F_OK;
}

int b2f_video_fetch(b2f_video *v, int64_t pair_index, void *host_flow, size_t step) {
    if (!v || !host_flow || pair_index < 0) return B2F_BAD_ARG;
    if (step < 8 * (size_t)v->cols) return B2F_BAD_ARG;
    b2f::DeviceScope dev(v->device);
    const int slot = static_cast<int>(pair_index % v->depth);
    if (v->flow_pair[slot] != pair_index) return B2F_BAD_ARG;  // not pushed yet, or already overwritten
    VCHECK(cudaEventSynchronize(v->down_done[slot]));
    const char *src = v->h_flow(pair_index);
    const size_t row_bytes = 8 * (size_t)v->cols;
    for (int y = 0; y < v->rows; ++y)
        std::memcpy(static_cast<char *>(host_flow) + (size_t)y * step, src + (size_t)y * row_bytes, row_bytes);
    return B2F_OK;
}

int b2f_video_fetch_view(b2f_video *v, int64_t pair_index, const float **host_flow, size_t *step) {
    if (!v || !host_flow || !step || pair_index < 0) return B2F_BAD_ARG;
    b2f::DeviceScope dev(v->device);
    const int slot = static_cast<int>(pair_index % v->depth);
    if (v->flow_pair[slot] != pair_index) return B2F_BAD_ARG;
    VCHECK(cudaEventSynchronize(v->down_done[slot]));
    *host_flow = reinterpret_cast<const float *>(v->h_flow(pair_index));
    *step = 8 * (size_t)v->cols;
    return B2F_OK;
}

}  // extern "C"
