// runtime.cu -- arena, launch context, handle base and the algorithm-independent part of the
// C ABI declared in include/b200flow.h.
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>

namespace b2f {

int cv_round(double v) { return static_cast<int>(std::nearbyint(v)); }  // FE_TONEAREST = half-even

// ------------------------------------------------------------------------------------ Arena
Arena::~Arena() { release(); }

void Arena::release() {
    if (base_) cudaFree(base_);
    base_ = nullptr;
    cap_ = 0;
}

cudaError_t Arena::reserve(size_t n) {
    if (n <= cap_) return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc(&base_, n);
    if (e != cudaSuccess) {
        base_ = nullptr;
        return e;
    }
    cap_ = n;
    return cudaSuccess;
}

void *Arena::bytes(size_t n) {
    size_t a = (off_ + 255) & ~size_t(255);
    off_ = a + n;
    if (counting_) return nullptr;
    return base_ + a;
}

Plane Arena::plane(int rows, int cols) {
    Plane pl;
    pl.pitch = plane_pitch(cols);
    // one extra row of slack so vectorised tails never leave the allocation
    pl.p = static_cast<float *>(bytes(sizeof(float) * (size_t)pl.pitch * (rows + 1)));
    return pl;
}

// ------------------------------------------------------------------------------------ Ctx
void Ctx::pre(int cls, double bytes) {
    if (stats) {
        stats->launches++;
        if (cls >= 0 && cls < B2F_MAX_KERNEL_CLASSES) {
            stats->class_launches[cls]++;
            stats->class_bytes[cls] += bytes;
        }
    }
    if (profiling && !capturing && timed && event_pool) {
        Timed t;
        t.cls = cls;
        auto get = [&]() {
            cudaEvent_t e = nullptr;
            if (!event_pool->empty()) {
                e = event_pool->back();
                event_pool->pop_back();
            } else {
                check(cudaEventCreate(&e));
            }
            return e;
        };
        t.e0 = get();
        t.e1 = get();
        check(cudaEventRecord(t.e0, stream));
        timed->push_back(t);
    }
}

void Ctx::post(int cls) {
    (void)cls;
    check(cudaPeekAtLastError());
    if (profiling && !capturing && timed && !timed->empty()) check(cudaEventRecord(timed->back().e1, stream));
}

}  // namespace b2f

// ------------------------------------------------------------------------------------ handle base
b2f_handle::~b2f_handle() {
    for (auto &t : timed) {
        cudaEventDestroy(t.e0);
        cudaEventDestroy(t.e1);
    }
    for (auto e : event_pool) cudaEventDestroy(e);
    if (host_stage) cudaFree(host_stage);
    if (ext_stage) cudaFree(ext_stage);
}

b2f::Ctx b2f_handle::make_ctx(cudaStream_t s) {
    b2f::Ctx c;
    c.stream = s;
    c.stats = &stats;
    c.profiling = profiling;
    c.timed = &timed;
    c.event_pool = &event_pool;
    return c;
}

int b2f_handle::sm_count() {
    if (!sm_count_) {
        int dev = device, n = 0;
        if ((dev >= 0 || cudaGetDevice(&dev) == cudaSuccess) &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) {
            sm_count_ = n;
        } else {
            cudaGetLastError();  // a failed query must not surface as the next launch's error
            sm_count_ = 132;
        }
    }
    return sm_count_;
}

int b2f_handle::finish(b2f::Ctx &ctx, cudaStream_t s) {
    if (ctx.ok() && s == nullptr) ctx.check(cudaDeviceSynchronize());  // legacy-stream contract
    if (!ctx.ok()) {
        last_cuda_error = static_cast<int>(ctx.err);
        cudaGetLastError();  // clear sticky-less error state
        return ctx.err == cudaErrorMemoryAllocation ? B2F_OUT_OF_MEMORY : B2F_CUDA_ERROR;
    }
    return B2F_OK;
}

void b2f_handle::collect_profile() {
    for (auto &t : timed) {
        if (cudaEventSynchronize(t.e1) == cudaSuccess) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess && t.cls >= 0 && t.cls < B2F_MAX_KERNEL_CLASSES)
                stats.class_ms[t.cls] += ms;
        }
        event_pool.push_back(t.e0);
        event_pool.push_back(t.e1);
    }
    timed.clear();
}

namespace {
// b2f_approx_probe: rcp_approx / sqrt_approx from common.cuh, the functions the TV-L1 kernels call, element-wise
__global__ void k_approx_probe(int op, const float *__restrict__ in, float *__restrict__ out, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = op == 0 ? b2f::rcp_approx(in[i]) : b2f::sqrt_approx(in[i]);
}
}  // namespace

// ------------------------------------------------------------------------------------ C ABI (generic part)
extern "C" {

int b2f_approx_probe(int op, const float *in, float *out, size_t n, void *cuda_stream) {
    if (!(op == 0 || op == 1) || (n && (!in || !out))) return B2F_BAD_ARG;
    if (n == 0) return B2F_OK;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    b2f::DeviceScope dev(in, s);
    const size_t blocks = std::min<size_t>((n + 255) / 256, 65535 * 8);
    k_approx_probe<<<(unsigned)blocks, 256, 0, s>>>(op, in, out, n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && s == nullptr) e = cudaDeviceSynchronize();
    return e == cudaSuccess ? B2F_OK : B2F_CUDA_ERROR;
}

void b2f_destroy(b2f_handle *h) { delete h; }

int b2f_set_param(b2f_handle *h, int id, double value) {
    if (!h) return B2F_BAD_ARG;
    switch (id) {
        case B2F_ENGINE_FUSED_ITERS: h->knobs.fused_iters = static_cast<int>(value); return B2F_OK;
        case B2F_ENGINE_USE_GRAPH: h->knobs.use_graph = value != 0; return B2F_OK;
        case B2F_ENGINE_KERNEL_PATH: h->knobs.kernel_path = static_cast<int>(value); return B2F_OK;
        case B2F_ENGINE_AUX_PATH: h->knobs.aux_path = static_cast<int>(value); return B2F_OK;
        default: return id >= B2F_ENGINE_ACTIVE_PATH ? B2F_BAD_ARG : h->set_param(id, value);  // active paths: read-only
    }
}

int b2f_get_param(const b2f_handle *h, int id, double *value) {
    if (!h || !value) return B2F_BAD_ARG;
    switch (id) {
        case B2F_ENGINE_FUSED_ITERS: *value = h->knobs.fused_iters; return B2F_OK;
        case B2F_ENGINE_USE_GRAPH: *value = h->knobs.use_graph; return B2F_OK;
        case B2F_ENGINE_KERNEL_PATH: *value = h->knobs.kernel_path; return B2F_OK;
        case B2F_ENGINE_AUX_PATH: *value = h->knobs.aux_path; return B2F_OK;
        default: break;
    }
    if (id < B2F_ENGINE_ACTIVE_PATH) return h->get_param(id, value);
    const int i = id - B2F_ENGINE_ACTIVE_PATH - h->active_path_first;  // a level the last calc did not solve: BAD_ARG
    if (i < 0 || i >= static_cast<int>(h->active_paths.size())) return B2F_BAD_ARG;
    *value = h->active_paths[i];
    return B2F_OK;
}

const char *b2f_default_name(const b2f_handle *h) { return h ? h->default_name() : ""; }

static int check_images(const b2f_image *I0, const b2f_image *I1, const b2f_image *flow) {
    if (!I0 || !I1 || !flow) return B2F_BAD_ARG;
    if (!I0->data || !I1->data || !flow->data) return B2F_BAD_ARG;
    if (I0->rows <= 0 || I0->cols <= 0) return B2F_BAD_ARG;
    return B2F_OK;
}

int b2f_calc(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *flow, void *cuda_stream) {
    if (!h) return B2F_BAD_ARG;
    int st = check_images(I0, I1, flow);
    if (st != B2F_OK) return st;
    h->stats.calls++;
    b2f::DeviceScope dev(I0->data, static_cast<cudaStream_t>(cuda_stream));
    if (!h->bind_device()) return B2F_BAD_ARG;
    return h->calc(I0, I1, flow, static_cast<cudaStream_t>(cuda_stream));
}

int b2f_calc_uv(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *u, b2f_image *v,
                void *cuda_stream) {
    if (!h || !v) return B2F_BAD_ARG;
    int st = check_images(I0, I1, u);
    if (st != B2F_OK) return st;
    if (!v->data) return B2F_BAD_ARG;
    if (u->type != B2F_32FC1 || v->type != B2F_32FC1) return B2F_UNSUPPORTED_TYPE;
    if (v->rows != u->rows || v->cols != u->cols) return B2F_SIZE_MISMATCH;
    h->stats.calls++;
    b2f::DeviceScope dev(I0->data, static_cast<cudaStream_t>(cuda_stream));
    if (!h->bind_device()) return B2F_BAD_ARG;
    h->planar_v = v->data;
    h->planar_v_step = v->step;
    st = h->calc(I0, I1, u, static_cast<cudaStream_t>(cuda_stream));
    h->planar_v = nullptr;
    h->planar_v_step = 0;
    return st;
}

static size_t elem_size(int type) {
    switch (type) {
        case B2F_8UC1: return 1;
        case B2F_32FC1: return 4;
        case B2F_32FC2: return 8;
        default: return 0;
    }
}

int b2f_calc_host(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *flow, void *cuda_stream) {
    if (!h) return B2F_BAD_ARG;
    int st = check_images(I0, I1, flow);
    if (st != B2F_OK) return st;
    size_t es = elem_size(I0->type), fs = elem_size(flow->type);
    if (es == 0 || I1->type != I0->type) return B2F_UNSUPPORTED_TYPE;
    if (fs != 8) return B2F_UNSUPPORTED_TYPE;
    if (I1->rows != I0->rows || I1->cols != I0->cols || flow->rows != I0->rows || flow->cols != I0->cols)
        return B2F_SIZE_MISMATCH;
    const int rows = I0->rows, cols = I0->cols;
    // a short pitch is a caller error, not a CUDA failure
    if (I0->step < cols * es || I1->step < cols * es || flow->step < cols * fs) return B2F_BAD_ARG;
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    b2f::DeviceScope dev(nullptr, s);  // host buffers: the stream names the device
    if (!h->bind_device()) return B2F_BAD_ARG;
    size_t in_pitch = (cols * es + 255) & ~size_t(255);
    size_t fl_pitch = (cols * fs + 255) & ~size_t(255);
    size_t need = 2 * in_pitch * rows + fl_pitch * rows;
    if (need > h->host_stage_bytes) {
        if (h->host_stage) cudaFree(h->host_stage);
        h->host_stage = nullptr;
        h->host_stage_bytes = 0;
        cudaError_t e = cudaMalloc(&h->host_stage, need);
        if (e != cudaSuccess) {
            h->last_cuda_error = e;
            cudaGetLastError();
            return B2F_OUT_OF_MEMORY;
        }
        h->host_stage_bytes = need;
    }
    char *d0 = static_cast<char *>(h->host_stage);
    char *d1 = d0 + in_pitch * rows;
    char *df = d1 + in_pitch * rows;
    cudaError_t e = cudaMemcpy2DAsync(d0, in_pitch, I0->data, I0->step, cols * es, rows, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess)
        e = cudaMemcpy2DAsync(d1, in_pitch, I1->data, I1->step, cols * es, rows, cudaMemcpyHostToDevice, s);
    b2f_image g0{d0, in_pitch, rows, cols, I0->type}, g1{d1, in_pitch, rows, cols, I1->type};
    b2f_image gf{df, fl_pitch, rows, cols, B2F_32FC2};
    if (e == cudaSuccess && h->reads_flow())  // only the use-initial-flow paths read the caller's flow (8 B/px of H2D)
        e = cudaMemcpy2DAsync(df, fl_pitch, flow->data, flow->step, cols * fs, rows, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
        h->last_cuda_error = e;
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    h->stats.calls++;
    st = h->calc(&g0, &g1, &gf, s);
    if (st != B2F_OK) return st;
    e = cudaMemcpy2DAsync(flow->data, flow->step, df, fl_pitch, cols * fs, rows, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        h->last_cuda_error = e;
        cudaGetLastError();
        return B2F_CUDA_ERROR;
    }
    return B2F_OK;
}

size_t b2f_workspace_bytes(b2f_handle *h, int rows, int cols, int type) {
    if (!h) return 0;
    if (rows <= 0 || cols <= 0) return h->arena.capacity();
    return h->workspace_bytes(rows, cols, type);
}

const char *b2f_status_string(int status) {
    switch (status) {
        case B2F_OK: return "B2F_OK";
        case B2F_BAD_ARG: return "B2F_BAD_ARG: invalid argument or parameter (reference: CV_Assert, StsAssert -215)";
        case B2F_UNSUPPORTED_TYPE: return "B2F_UNSUPPORTED_TYPE: image type not accepted by this algorithm";
        case B2F_SIZE_MISMATCH: return "B2F_SIZE_MISMATCH: I0, I1 and flow must have the same size";
        case B2F_CUDA_ERROR: return "B2F_CUDA_ERROR: CUDA runtime failure (reference: GpuApiCallError)";
        case B2F_NO_DEVICE: return "B2F_NO_DEVICE: no CUDA device (reference: throw_no_cuda)";
        case B2F_OUT_OF_MEMORY: return "B2F_OUT_OF_MEMORY";
        default: return "B2F_UNKNOWN_STATUS";
    }
}

int b2f_last_cuda_error(const b2f_handle *h) { return h ? h->last_cuda_error : 0; }

const char *b2f_version(void) { return "b200flow 0.1 (sm_90a)"; }

int b2f_get_stats(b2f_handle *h, b2f_stats *out) {
    if (!h || !out) return B2F_BAD_ARG;
    h->collect_profile();
    h->refresh_stats();
    *out = h->stats;
    return B2F_OK;
}

int b2f_reset_stats(b2f_handle *h) {
    if (!h) return B2F_BAD_ARG;
    h->collect_profile();
    int levels = h->stats.levels, it = h->stats.iterations_run;
    std::memset(&h->stats, 0, sizeof(h->stats));
    h->stats.levels = levels;
    h->stats.iterations_run = it;
    return B2F_OK;
}

const char *b2f_kernel_class_name(const b2f_handle *h, int cls) { return h ? h->class_name(cls) : ""; }

int b2f_set_profiling(b2f_handle *h, int on) {
    if (!h) return B2F_BAD_ARG;
    h->profiling = on != 0;
    return B2F_OK;
}

}  // extern "C"
