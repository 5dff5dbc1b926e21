// comm.cu -- native result gather of the batched front end (SURVEY.md 8b "b2f_batch_run(..., ncclComm_t)", 8e).
//
// Frame pairs are independent, so the ONLY exchange of the multi-GPU path is the gather of the finished CV_32FC2
// fields to one rank.  Round 1 did it in Python with one torch.distributed.gather per step, after the whole batch:
// rank 0 ingested (N-1) x 32 x 16.6 MB serially at the end of every step (0.966 scaling efficiency at N = 8).
// Here every pair is sent as soon as ITS solve finishes: the engine stream records an event, a dedicated
// communication stream waits for it and issues ncclSend (non-root) / the matching group of ncclRecv (root), so the
// transfers of pair i overlap the solves of pairs i+1.. and only the last pair's transfer is exposed.
//
// NCCL is not linked: the symbols are taken from the libnccl.so.2 already loaded in the process (torch's) or, failing
// that, from the system library, through dlopen -- libb200flow.so keeps loading on machines without NCCL and the
// single-GPU path never touches it.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>
#include <new>
#include <vector>

#include <climits>
#include "common.cuh"

struct b2f_batch;
namespace b2f {
// batch.cu
int batch_run_device_impl(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1, b2f_image *flow,
                          cudaStream_t cur, struct b2f_comm *comm, int dst, b2f_image *gathered);
}  // namespace b2f

namespace {

struct NcclApi {
    void *lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitRankConfig)(ncclComm_t *, int, ncclUniqueId, int, void *) = nullptr;  // optional (>= 2.14)
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*CommCount)(const ncclComm_t, int *) = nullptr;
    ncclResult_t (*CommUserRank)(const ncclComm_t, int *) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    bool ok = false;
};

NcclApi *nccl_api() {
    static NcclApi api = [] {  // a function-local static is initialised once, thread-safely
        NcclApi a;
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // the copy torch already loaded, if any
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return a;
        a.lib = h;
#define B2F_SYM(field, name) *reinterpret_cast<void **>(&a.field) = dlsym(h, name)
        B2F_SYM(GetUniqueId, "ncclGetUniqueId");
        B2F_SYM(CommInitRank, "ncclCommInitRank");
        B2F_SYM(CommInitRankConfig, "ncclCommInitRankConfig");
        B2F_SYM(CommDestroy, "ncclCommDestroy");
        B2F_SYM(CommCount, "ncclCommCount");
        B2F_SYM(CommUserRank, "ncclCommUserRank");
        B2F_SYM(Send, "ncclSend");
        B2F_SYM(Recv, "ncclRecv");
        B2F_SYM(GroupStart, "ncclGroupStart");
        B2F_SYM(GroupEnd, "ncclGroupEnd");
#undef B2F_SYM
        a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.CommCount && a.CommUserRank && a.Send && a.Recv &&
               a.GroupStart && a.GroupEnd;
        return a;
    }();
    return api.ok ? &api : nullptr;
}

}  // namespace

struct b2f_comm {
    NcclApi *api = nullptr;
    ncclComm_t comm = nullptr;
    bool owns = false;
    int rank = 0, nranks = 1, device = 0;
    cudaStream_t stream = nullptr;  // communication stream
    cudaEvent_t done = nullptr;
    std::vector<cudaEvent_t> pair_done;  // one per pair of the largest batch seen
    int last_nccl_error = 0;
};

namespace b2f {

// called by batch.cu after pair i was enqueued on engine stream `es`: order the transfer of that flow behind it
int comm_enqueue_pair(b2f_comm *c, int i, int n_pairs, cudaStream_t es, const b2f_image *flow_i, int dst,
                      b2f_image *gathered) {
    if (c->nranks == 1) return B2F_OK;
    while ((int)c->pair_done.size() <= i) {
        cudaEvent_t e = nullptr;
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) {
            cudaGetLastError();
            return B2F_CUDA_ERROR;
        }
        c->pair_done.push_back(e);
    }
    const size_t count = (size_t)flow_i->rows * flow_i->cols * 2;
    auto nccl_ok = [&](ncclResult_t r) {
        if (r != ncclSuccess) c->last_nccl_error = (int)r;
        return r == ncclSuccess;
    };
    if (c->rank != dst) {
        if (flow_i->step != (size_t)flow_i->cols * 8) return B2F_BAD_ARG;  // one contiguous message per flow
        if (cudaEventRecord(c->pair_done[i], es) != cudaSuccess || cudaStreamWaitEvent(c->stream, c->pair_done[i], 0) != cudaSuccess) {
            cudaGetLastError();
            return B2F_CUDA_ERROR;
        }
        if (!nccl_ok(c->api->Send(flow_i->data, count, ncclFloat, dst, c->comm, c->stream))) return B2F_CUDA_ERROR;
        return B2F_OK;
    }
    // root: the receives of pair i do not depend on the local solve, but they are ordered behind it all the same.
    // An NCCL receive is a kernel that spins on an SM until its peer sends; posted at batch start it would hold
    // that SM for the whole batch.  Behind the root's own pair i it starts about when the peers (which run in
    // lock step) start sending theirs.
    if (!gathered) return B2F_BAD_ARG;
    if (cudaEventRecord(c->pair_done[i], es) != cudaSuccess || cudaStreamWaitEvent(c->stream, c->pair_done[i], 0) != cudaSuccess) {
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    if (!nccl_ok(c->api->GroupStart())) return B2F_CUDA_ERROR;
    bool ok = true;
    for (int r = 0; r < c->nranks && ok; ++r) {
        if (r == dst) continue;
        const b2f_image &g = gathered[(size_t)r * n_pairs + i];
        if (!g.data || g.rows != flow_i->rows || g.cols != flow_i->cols || g.step != (size_t)g.cols * 8) {
            ok = false;
            break;
        }
        ok = nccl_ok(c->api->Recv(g.data, count, ncclFloat, r, c->comm, c->stream));
    }
    const bool ended = nccl_ok(c->api->GroupEnd());
    if (!ok || !ended) return ok ? B2F_CUDA_ERROR : B2F_BAD_ARG;
    // own flow: straight into its slot unless the caller already pointed flow[i] there
    const b2f_image &mine = gathered[(size_t)dst * n_pairs + i];
    if (mine.data && mine.data != flow_i->data) {
        if (mine.rows != flow_i->rows || mine.cols != flow_i->cols) return B2F_BAD_ARG;
        if (cudaMemcpy2DAsync(mine.data, mine.step, flow_i->data, flow_i->step, (size_t)flow_i->cols * 8, flow_i->rows,
                              cudaMemcpyDeviceToDevice, es) != cudaSuccess) {
            cudaGetLastError();
            return B2F_CUDA_ERROR;
        }
    }
    return B2F_OK;
}

// join: the caller's stream continues after every transfer of this batch
int comm_join(b2f_comm *c, cudaStream_t cur) {
    if (c->nranks == 1) return B2F_OK;
    if (cudaEventRecord(c->done, c->stream) != cudaSuccess || cudaStreamWaitEvent(cur, c->done, 0) != cudaSuccess) {
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    return B2F_OK;
}

// fork: transfers of this batch start after whatever the caller enqueued before it (e.g. the previous batch's consumers)
int comm_fork(b2f_comm *c, cudaEvent_t start) {
    if (c->nranks == 1) return B2F_OK;
    if (cudaStreamWaitEvent(c->stream, start, 0) != cudaSuccess) {
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    return B2F_OK;
}

int comm_device(const b2f_comm *c) { return c->device; }

}  // namespace b2f

extern "C" {

int b2f_comm_available(void) { return nccl_api() != nullptr; }

int b2f_comm_unique_id(void *id, size_t bytes) {
    NcclApi *api = nccl_api();
    if (!api) return B2F_NO_DEVICE;
    if (!id || bytes < sizeof(ncclUniqueId)) return B2F_BAD_ARG;
    ncclUniqueId u;
    if (api->GetUniqueId(&u) != ncclSuccess) return B2F_CUDA_ERROR;
    std::memcpy(id, &u, sizeof(u));
    return B2F_OK;
}

static int finish_create(b2f_comm *c, b2f_comm **out) {
    // highest priority: a transfer's CTA is placed as soon as any solver CTA retires
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (cudaGetDevice(&c->device) != cudaSuccess ||
        cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming) != cudaSuccess) {
        cudaGetLastError();
        b2f_comm_destroy(c);
        return B2F_CUDA_ERROR;
    }
    *out = c;
    return B2F_OK;
}

int b2f_comm_create(const void *id, size_t bytes, int rank, int nranks, b2f_comm **out) {
    if (!out || nranks < 1 || rank < 0 || rank >= nranks) return B2F_BAD_ARG;
    *out = nullptr;
    b2f_comm *c = new (std::nothrow) b2f_comm;
    if (!c) return B2F_OUT_OF_MEMORY;
    c->rank = rank;
    c->nranks = nranks;
    if (nranks > 1) {
        NcclApi *api = nccl_api();
        if (!api) { delete c; return B2F_NO_DEVICE; }
        if (!id || bytes < sizeof(ncclUniqueId)) { delete c; return B2F_BAD_ARG; }
        ncclUniqueId u;
        std::memcpy(&u, id, sizeof(u));
        c->api = api;
        // A flow is 16.6 MB and a rank produces on the order of a hundred of them a second: one channel per pair of
        // ranks is plenty (four when the root takes in seven peers), and every further NCCL CTA would sit on an SM the
        // solvers want.  The config layout is NCCL 2.17's; newer libraries
        // accept it by its size/version fields.
        struct CommConfig217 {
            size_t size;
            unsigned magic, version;
            int blocking, cga_cluster_size, min_ctas, max_ctas;
            const char *net_name;
            int split_share;
        } cfg = {sizeof(CommConfig217), 0xcafebeefu, 21700u, INT_MIN, INT_MIN, 1, nranks <= 2 ? 1 : 4, nullptr, INT_MIN};
        ncclResult_t r = ncclInvalidUsage;
        if (api->CommInitRankConfig) r = api->CommInitRankConfig(&c->comm, nranks, u, rank, &cfg);
        if (r != ncclSuccess) r = api->CommInitRank(&c->comm, nranks, u, rank);  // collective: every rank calls it
        if (r != ncclSuccess) {
            c->last_nccl_error = (int)r;
            delete c;
            return B2F_CUDA_ERROR;
        }
        c->owns = true;
    }
    return finish_create(c, out);
}

int b2f_comm_adopt(void *nccl_comm, b2f_comm **out) {
    if (!out || !nccl_comm) return B2F_BAD_ARG;
    *out = nullptr;
    NcclApi *api = nccl_api();
    if (!api) return B2F_NO_DEVICE;
    b2f_comm *c = new (std::nothrow) b2f_comm;
    if (!c) return B2F_OUT_OF_MEMORY;
    c->api = api;
    c->comm = static_cast<ncclComm_t>(nccl_comm);
    if (api->CommCount(c->comm, &c->nranks) != ncclSuccess || api->CommUserRank(c->comm, &c->rank) != ncclSuccess) {
        delete c;
        return B2F_BAD_ARG;
    }
    return finish_create(c, out);
}

void b2f_comm_destroy(b2f_comm *c) {
    if (!c) return;
    b2f::DeviceScope dev(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->owns && c->comm && c->api) c->api->CommDestroy(c->comm);
    for (auto e : c->pair_done)
        if (e) cudaEventDestroy(e);
    if (c->done) cudaEventDestroy(c->done);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

int b2f_comm_rank(const b2f_comm *c) { return c ? c->rank : -1; }
int b2f_comm_nranks(const b2f_comm *c) { return c ? c->nranks : 0; }
int b2f_comm_last_nccl_error(const b2f_comm *c) { return c ? c->last_nccl_error : 0; }

int b2f_batch_run_device_gather(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1, b2f_image *flow,
                                b2f_comm *comm, int dst, b2f_image *gathered, void *cuda_stream) {
    if (!comm || dst < 0 || dst >= comm->nranks) return B2F_BAD_ARG;
    return b2f::batch_run_device_impl(b, n_pairs, I0, I1, flow, static_cast<cudaStream_t>(cuda_stream), comm, dst, gathered);
}

}  // extern "C"
