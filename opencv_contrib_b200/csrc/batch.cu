// batch.cu -- native batched frame-pair front end for ONE GPU (SURVEY.md 8b "b2f_batch_run", 8e).
//
// Frame pairs are independent problems and engine instances are not re-entrant (they cache buffers, like the
// reference's: tvl1flow.cpp:141-167), so a batch owns N engine handles on N CUDA streams and deals the pairs
// round robin -- the shape of the reference's own multi-stream test (test_optflow.cpp:468-528).  Independent
// pairs fill each other's launch-bound coarse levels and pipeline tails.
//   * run_device: inputs / outputs resident; the work is forked from and joined to the caller's stream with
//     events only, so CUDA events on that stream bracket the whole batch and nothing blocks the host;
//   * run_host: one worker thread per stream uploads, solves and downloads its share through b2f_calc_host, so
//     the copies of one pair overlap the solves of the others; returns when every flow is in host memory.
// Sharding across GPUs is one process per GPU (rank r owns a contiguous block of pairs); the result gather to one rank
// is native too: b2f_batch_run_device_gather sends every flow over NCCL as soon as its solve finishes (comm.cu).
#include <atomic>
#include <new>
#include <thread>
#include <vector>

#include "common.cuh"

struct b2f_batch {
    int device = 0;
    std::vector<b2f_handle *> engines;
    std::vector<cudaStream_t> streams;
    std::vector<cudaEvent_t> done;
    cudaEvent_t start = nullptr;
    int last_status = B2F_OK;
};

struct b2f_comm;
namespace b2f {
// comm.cu
int comm_enqueue_pair(b2f_comm *c, int i, int n_pairs, cudaStream_t es, const b2f_image *flow_i, int dst, b2f_image *gathered);
int comm_fork(b2f_comm *c, cudaEvent_t start);
int comm_join(b2f_comm *c, cudaStream_t cur);
int comm_device(const b2f_comm *c);

int batch_run_device_impl(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1, b2f_image *flow,
                          cudaStream_t cur, b2f_comm *comm, int dst, b2f_image *gathered) {
    if (!b || n_pairs < 0 || (n_pairs > 0 && (!I0 || !I1 || !flow))) return B2F_BAD_ARG;
    if (n_pairs == 0) return B2F_OK;
    if (comm && comm_device(comm) != b->device) return B2F_BAD_ARG;
    DeviceScope dev(b->device);
    const int ns = static_cast<int>(b->streams.size());
    const int used = n_pairs < ns ? n_pairs : ns;
    auto fail = [&]() {
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    };
    if (cudaEventRecord(b->start, cur) != cudaSuccess) return fail();
    for (int k = 0; k < used; ++k)
        if (cudaStreamWaitEvent(b->streams[k], b->start, 0) != cudaSuccess) return fail();
    int status = comm ? comm_fork(comm, b->start) : B2F_OK;
    for (int i = 0; i < n_pairs && status == B2F_OK; ++i) {
        const int k = i % ns;
        status = b2f_calc(b->engines[k], &I0[i], &I1[i], &flow[i], b->streams[k]);
        if (status == B2F_OK && comm) status = comm_enqueue_pair(comm, i, n_pairs, b->streams[k], &flow[i], dst, gathered);
    }
    // join even after a failure so the caller's stream stays ordered behind whatever was enqueued
    for (int k = 0; k < used; ++k) {
        if (cudaEventRecord(b->done[k], b->streams[k]) != cudaSuccess) return fail();
        if (cudaStreamWaitEvent(cur, b->done[k], 0) != cudaSuccess) return fail();
    }
    if (comm) {
        const int js = comm_join(comm, cur);
        if (status == B2F_OK) status = js;
    }
    if (status == B2F_OK && cur == nullptr && cudaDeviceSynchronize() != cudaSuccess) return fail();
    b->last_status = status;
    return status;
}
}  // namespace b2f

extern "C" {

void b2f_batch_destroy(b2f_batch *b) {
    if (!b) return;
    b2f::DeviceScope dev(b->device);
    for (auto s : b->streams)
        if (s) cudaStreamSynchronize(s);
    for (auto h : b->engines) b2f_destroy(h);
    for (auto e : b->done)
        if (e) cudaEventDestroy(e);
    if (b->start) cudaEventDestroy(b->start);
    for (auto s : b->streams)
        if (s) cudaStreamDestroy(s);
    delete b;
}

int b2f_batch_create(int algo, const void *params, int n_streams, b2f_batch **out) {
    if (!out || n_streams < 1 || n_streams > 64) return B2F_BAD_ARG;
    *out = nullptr;
    b2f_batch *b = new (std::nothrow) b2f_batch;
    if (!b) return B2F_OUT_OF_MEMORY;
    if (cudaGetDevice(&b->device) != cudaSuccess) {
        cudaGetLastError();
        delete b;
        return B2F_NO_DEVICE;
    }
    int st = B2F_OK;
    for (int i = 0; i < n_streams && st == B2F_OK; ++i) {
        b2f_handle *h = nullptr;
        switch (algo) {
            case b2f::ALGO_TVL1: st = b2f_tvl1_create(static_cast<const b2f_tvl1_params *>(params), &h); break;
            case b2f::ALGO_FARNEBACK: st = b2f_farneback_create(static_cast<const b2f_farneback_params *>(params), &h); break;
            case b2f::ALGO_BROX: st = b2f_brox_create(static_cast<const b2f_brox_params *>(params), &h); break;
            case b2f::ALGO_DENSELK: st = b2f_denselk_create(static_cast<const b2f_denselk_params *>(params), &h); break;
            case b2f::ALGO_DEEPFLOW: st = b2f_deepflow_create(static_cast<const b2f_deepflow_params *>(params), &h); break;
            case b2f::ALGO_DIS: st = b2f_dis_create(static_cast<const b2f_dis_params *>(params), &h); break;
            case b2f::ALGO_FASTBM: st = b2f_fastbm_create(static_cast<const b2f_fastbm_params *>(params), &h); break;
            case b2f::ALGO_VARREF: st = b2f_varref_create(static_cast<const b2f_varref_params *>(params), &h); break;
            case b2f::ALGO_OPTFLOWGF: st = b2f_optflowgf_create(static_cast<const b2f_farneback_params *>(params), &h); break;
            default: st = B2F_BAD_ARG;
        }
        if (st != B2F_OK) break;
        b->engines.push_back(h);
        cudaStream_t s = nullptr;
        cudaEvent_t e = nullptr;
        if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) {
            cudaGetLastError();
            if (s) cudaStreamDestroy(s);
            st = B2F_CUDA_ERROR;
            break;
        }
        b->streams.push_back(s);
        b->done.push_back(e);
    }
    if (st == B2F_OK && cudaEventCreateWithFlags(&b->start, cudaEventDisableTiming) != cudaSuccess) {
        cudaGetLastError();
        st = B2F_CUDA_ERROR;
    }
    if (st != B2F_OK) {
        b2f_batch_destroy(b);
        return st;
    }
    *out = b;
    return B2F_OK;
}

int b2f_batch_streams(const b2f_batch *b) { return b ? static_cast<int>(b->streams.size()) : 0; }

b2f_handle *b2f_batch_engine(b2f_batch *b, int i) {
    return (b && i >= 0 && i < static_cast<int>(b->engines.size())) ? b->engines[i] : nullptr;
}

int b2f_batch_set_param(b2f_batch *b, int id, double value) {
    if (!b) return B2F_BAD_ARG;
    for (auto h : b->engines) {
        const int st = b2f_set_param(h, id, value);
        if (st != B2F_OK) return st;
    }
    return B2F_OK;
}

int b2f_batch_run_device(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1, b2f_image *flow,
                         void *cuda_stream) {
    return b2f::batch_run_device_impl(b, n_pairs, I0, I1, flow, static_cast<cudaStream_t>(cuda_stream), nullptr, 0, nullptr);
}

int b2f_batch_run_host(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1, b2f_image *flow) {
    if (!b || n_pairs < 0 || (n_pairs > 0 && (!I0 || !I1 || !flow))) return B2F_BAD_ARG;
    if (n_pairs == 0) return B2F_OK;
    const int ns = static_cast<int>(b->streams.size());
    const int used = n_pairs < ns ? n_pairs : ns;
    std::atomic<int> status{B2F_OK};
    auto work = [&](int k) {
        b2f::DeviceScope dev(b->device);  // the current device is per thread
        for (int i = k; i < n_pairs; i += ns) {
            if (status.load() != B2F_OK) return;
            const int st = b2f_calc_host(b->engines[k], &I0[i], &I1[i], &flow[i], b->streams[k]);
            if (st != B2F_OK) {
                int expected = B2F_OK;
                status.compare_exchange_strong(expected, st);
                return;
            }
        }
    };
    std::vector<std::thread> threads;
    threads.reserve(used);
    for (int k = 1; k < used; ++k) threads.emplace_back(work, k);
    work(0);
    for (auto &t : threads) t.join();
    b->last_status = status.load();
    return b->last_status;
}

uint64_t b2f_batch_launches(b2f_batch *b) {
    if (!b) return 0;
    uint64_t n = 0;
    for (auto h : b->engines) n += h->stats.launches;
    return n;
}

int b2f_batch_reset_stats(b2f_batch *b) {
    if (!b) return B2F_BAD_ARG;
    for (auto h : b->engines) b2f_reset_stats(h);
    return B2F_OK;
}

}  // extern "C"
