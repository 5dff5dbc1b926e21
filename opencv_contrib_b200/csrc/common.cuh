// common.cuh -- shared host/device plumbing for libb200flow (sm_90a only).
//
// Engine conventions:
//  * every work plane is float32, row-major, pitch (in floats) a multiple of 32 so rows start on
//    128-byte lines and are float4-loadable / TMA-addressable;
//  * one arena (single cudaMalloc) per handle, laid out once per (rows, cols, params);
//  * all kernels run on the caller's stream; no global mutable device state (__constant__
//    symbols) so handles never interfere (the reference's global tables -- farneback.cu:60-63,
//    pyrlk.cu:60-64 -- make concurrent instances race; SURVEY.md §7).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <float.h>
#include <atomic>
#include <vector>
#include <string>

#include "b200flow.h"

namespace b2f {

// ---------------------------------------------------------------------------------------------
// Plane views
// ---------------------------------------------------------------------------------------------
struct Plane {
    float *p;
    int pitch;  // floats
    __host__ __device__ __forceinline__ float &at(int y, int x) const { return p[(size_t)y * pitch + x]; }
    __host__ __device__ __forceinline__ float *row(int y) const { return p + (size_t)y * pitch; }
};

// Caller-provided image (possibly an ROI with arbitrary byte pitch).
struct ImageView {
    void *data;
    size_t step;  // bytes
    int rows, cols, type;
    void *data2 = nullptr;  // planar flow output (b2f_calc_uv): data = u plane, data2 = v plane
    size_t step2 = 0;
};

static inline int round_up(int v, int m) { return (v + m - 1) / m * m; }
static inline int div_up(int a, int b) { return (a + b - 1) / b; }
static inline int plane_pitch(int cols) { return round_up(cols, 32); }

// cvRound / saturate_cast<int>(double): round half to even (SURVEY.md §9.2).
int cv_round(double v);

// ---------------------------------------------------------------------------------------------
// Arena: bump allocator over one device allocation
// ---------------------------------------------------------------------------------------------
class Arena {
public:
    ~Arena();
    // Two-phase use: begin(true) + alloc... = counting pass; reserve(); begin(false) + alloc... again.
    void begin(bool counting) { counting_ = counting; off_ = 0; }
    Plane plane(int rows, int cols);
    void *bytes(size_t n);
    size_t used() const { return off_; }
    size_t capacity() const { return cap_; }
    cudaError_t reserve(size_t n);  // (re)allocates when n > capacity
    void release();

private:
    char *base_ = nullptr;
    size_t cap_ = 0, off_ = 0;
    bool counting_ = true;
};

// ---------------------------------------------------------------------------------------------
// Launch context: stream + accounting + optional per-launch event timing
// ---------------------------------------------------------------------------------------------
struct Ctx {
    cudaStream_t stream = nullptr;
    b2f_stats *stats = nullptr;
    bool profiling = false;
    bool capturing = false;  // inside stream capture: no events, no error polling that syncs
    cudaError_t err = cudaSuccess;
    struct Timed { int cls; cudaEvent_t e0, e1; };
    std::vector<Timed> *timed = nullptr;      // filled while profiling
    std::vector<cudaEvent_t> *event_pool = nullptr;

    void pre(int cls, double bytes);
    void post(int cls);
    bool ok() const { return err == cudaSuccess; }
    void check(cudaError_t e) { if (err == cudaSuccess && e != cudaSuccess) err = e; }
};

#define B2F_LAUNCH(ctx, cls, bytes, kernel, grid, block, smem, ...)                    \
    do {                                                                                \
        if ((ctx).ok()) {                                                               \
            (ctx).pre((cls), (bytes));                                                  \
            kernel<<<(grid), (block), (smem), (ctx).stream>>>(__VA_ARGS__);             \
            (ctx).post((cls));                                                          \
        }                                                                               \
    } while (0)

// ---------------------------------------------------------------------------------------------
// Device scope: the CUDA current device is per host thread.  A caller that drives several GPUs (or one GPU
// from worker threads that never called cudaSetDevice) passes a stream / device pointers of device N while
// the thread's current device is still 0; every entry point therefore switches to the device that owns the
// stream (or, for the NULL stream, the input image) for the duration of the call and restores it afterwards.
// The reference leaves this to the caller (cv::cuda::setDevice per thread).
// ---------------------------------------------------------------------------------------------
struct DeviceScope {
    int prev = -1;
    bool switched = false;
    DeviceScope(const void *device_ptr, cudaStream_t s) {
        int target = -1;
        // cudaStreamGetDevice on a stream that is being captured fails and invalidates the capture: under capture
        // the device is taken from the image instead
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        if (s != nullptr && s != cudaStreamLegacy && s != cudaStreamPerThread && cudaStreamIsCapturing(s, &cap) != cudaSuccess) {
            cudaGetLastError();
            cap = cudaStreamCaptureStatusNone;
        }
        if (s != nullptr && s != cudaStreamLegacy && s != cudaStreamPerThread && cap == cudaStreamCaptureStatusNone) {
            if (cudaStreamGetDevice(s, &target) != cudaSuccess) {
                cudaGetLastError();
                target = -1;
            }
        }
        if (target < 0 && device_ptr) {
            cudaPointerAttributes a;
            if (cudaPointerGetAttributes(&a, device_ptr) == cudaSuccess &&
                (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged))
                target = a.device;
            else
                cudaGetLastError();
        }
        enter(target);
    }
    explicit DeviceScope(int target) { enter(target); }
    ~DeviceScope() {
        if (switched) cudaSetDevice(prev);
    }
    DeviceScope(const DeviceScope &) = delete;
    DeviceScope &operator=(const DeviceScope &) = delete;

private:
    void enter(int target) {
        if (target >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != target) switched = cudaSetDevice(target) == cudaSuccess;
    }
};

// ---------------------------------------------------------------------------------------------
// Handle base
// ---------------------------------------------------------------------------------------------
enum Algo { ALGO_TVL1 = 1, ALGO_FARNEBACK = 2, ALGO_BROX = 3, ALGO_DENSELK = 4, ALGO_DEEPFLOW = 5, ALGO_DIS = 6, ALGO_FASTBM = 7,
           ALGO_VARREF = 8, ALGO_OPTFLOWGF = 9 };

struct EngineKnobs {
    int fused_iters = 0;  // 0 = auto
    int use_graph = 1;
    int kernel_path = 0;  // 0 auto, 1 unfused reference-shaped kernels
    int aux_path = 0;     // variant of the secondary kernels (TV-L1 warp: 0 tiled / TMA-staged, 3 separable)
};

// Field-wise equality of the public parameter structs (they contain padding after int members, so memcmp on
// copies may see indeterminate bytes and miss a cache hit).
static inline bool same_params(const b2f_tvl1_params &a, const b2f_tvl1_params &b) {
    return a.tau == b.tau && a.lambda == b.lambda && a.theta == b.theta && a.nscales == b.nscales && a.warps == b.warps &&
           a.epsilon == b.epsilon && a.iterations == b.iterations && a.scale_step == b.scale_step && a.gamma == b.gamma &&
           a.use_initial_flow == b.use_initial_flow;
}
static inline bool same_params(const b2f_farneback_params &a, const b2f_farneback_params &b) {
    return a.num_levels == b.num_levels && a.pyr_scale == b.pyr_scale && a.fast_pyramids == b.fast_pyramids &&
           a.win_size == b.win_size && a.num_iters == b.num_iters && a.poly_n == b.poly_n && a.poly_sigma == b.poly_sigma &&
           a.flags == b.flags;
}
static inline bool same_params(const b2f_brox_params &a, const b2f_brox_params &b) {
    return a.alpha == b.alpha && a.gamma == b.gamma && a.scale_factor == b.scale_factor &&
           a.inner_iterations == b.inner_iterations && a.outer_iterations == b.outer_iterations &&
           a.solver_iterations == b.solver_iterations;
}
static inline bool same_knobs(const EngineKnobs &a, const EngineKnobs &b) {
    return a.fused_iters == b.fused_iters && a.use_graph == b.use_graph && a.kernel_path == b.kernel_path &&
           a.aux_path == b.aux_path;
}

}  // namespace b2f

struct b2f_handle {
    int algo = 0;
    int last_cuda_error = 0;
    // A handle belongs to the device of its first call (arena, CUDA graph, TMA descriptors and the SM count are
    // created there): a later call whose stream / images live on another device is refused with B2F_BAD_ARG.
    int device = -1;
    bool bind_device() {
        int cur = -1;
        if (cudaGetDevice(&cur) != cudaSuccess) { cudaGetLastError(); return true; }
        if (device < 0) device = cur;
        return device == cur;
    }
    b2f_stats stats{};
    bool profiling = false;
    b2f::EngineKnobs knobs;
    b2f::Arena arena;
    std::vector<b2f::Ctx::Timed> timed;
    std::vector<cudaEvent_t> event_pool;
    // planar flow output requested by b2f_calc_uv for the duration of one calc()
    void *planar_v = nullptr;
    size_t planar_v_step = 0;
    bool flow_type_ok(const b2f_image *flow) const {
        return planar_v ? flow->type == B2F_32FC1 : flow->type == B2F_32FC2;
    }
    bool flow_step_ok(const b2f_image *flow) const {
        const size_t row = (size_t)flow->cols * (planar_v ? 4 : 8);
        return flow->step >= row && (!planar_v || planar_v_step >= row);
    }
    b2f::ImageView flow_view(const b2f_image *flow, int rows, int cols) const {
        b2f::ImageView v{flow->data, flow->step, rows, cols, planar_v ? B2F_32FC1 : B2F_32FC2};
        v.data2 = planar_v;
        v.step2 = planar_v_step;
        return v;
    }
    // staging for b2f_calc_host
    void *host_stage = nullptr;
    size_t host_stage_bytes = 0;
    // work-type frames of b2f_calc_ext
    void *ext_stage = nullptr;
    size_t ext_stage_bytes = 0;

    virtual ~b2f_handle();
    virtual int calc(const b2f_image *I0, const b2f_image *I1, b2f_image *flow, cudaStream_t s) = 0;
    virtual int set_param(int id, double v) = 0;
    virtual int get_param(int id, double *v) const = 0;
    virtual const char *default_name() const = 0;
    virtual const char *class_name(int cls) const = 0;
    virtual size_t workspace_bytes(int rows, int cols, int type) = 0;
    // does calc() read the caller's `flow` before writing it (useInitialFlow / OPTFLOW_USE_INITIAL_FLOW)?
    virtual bool reads_flow() const { return false; }
    // statistics that live on the device until the caller's stream has been synchronised (b2f_get_stats calls this)
    virtual void refresh_stats() {}

    // What the last calc ran on each solved level, finest first: b2f_get_param answers B2F_ENGINE_ACTIVE_PATH +
    // active_path_first + i with active_paths[i].  Engines fill it in their schedule; a graph replay restores it.
    std::vector<double> active_paths;
    int active_path_first = 0;
    // SM count of the handle's device, queried once (132, the H100 SXM's, when the query fails)
    int sm_count();
    int sm_count_ = 0;

    b2f::Ctx make_ctx(cudaStream_t s);
    int finish(b2f::Ctx &ctx, cudaStream_t s);  // maps ctx.err -> status, NULL-stream sync
    void collect_profile();
};

namespace b2f {

// ---------------------------------------------------------------------------------------------
// Per-device one-time setup (kernel attributes) that any host thread may reach first.  run() calls `init`, which
// reports through c.check, unless it already succeeded on the current device; a failure is retried by the next call.
// ---------------------------------------------------------------------------------------------
class DeviceOnce {
public:
    template <class Init>
    void run(Ctx &c, Init &&init) {
        int dev = -1;
        c.check(cudaGetDevice(&dev));
        if (!c.ok()) return;
        const bool tracked = dev >= 0 && dev < kMaxDevices;
        if (tracked && done_[dev].load(std::memory_order_acquire)) return;
        init();
        if (tracked && c.ok()) done_[dev].store(true, std::memory_order_release);
    }

private:
    static constexpr int kMaxDevices = 64;
    std::atomic<bool> done_[kMaxDevices] = {};
};

// ---------------------------------------------------------------------------------------------
// CUDA-graph cache of a fixed launch schedule (one per handle).  run() replays the graph when `key` equals the key it
// was captured under.  Otherwise it records whatever `body` launches through the Ctx it is given -- on a private
// capture stream -- and keeps the graph and the key only when the capture succeeded.  The key names everything the
// schedule bakes in, the arena base included.  The capture's launch / byte accounting and the handle's active paths are
// remembered, so a replay updates b2f_stats and active_paths exactly like the eager path would.
// ---------------------------------------------------------------------------------------------
template <class Key>
class GraphCache {
public:
    ~GraphCache() { destroy(); }
    void destroy() {
        if (exec_) cudaGraphExecDestroy(exec_);
        exec_ = nullptr;
    }
    // true when the graph ran on `s`; the active paths are restored only then
    template <class Body>
    bool run(b2f_handle &h, Ctx &c, cudaStream_t s, const Key &key, Body &&body) {
        if (!c.ok()) return false;
        if (!exec_ || !(key_ == key)) {
            capture(h, c, body);
            if (!c.ok()) return false;
            key_ = key;
        }
        c.check(cudaGraphLaunch(exec_, s));
        h.stats.launches += launches_;
        for (int i = 0; i < B2F_MAX_KERNEL_CLASSES; ++i) {
            h.stats.class_launches[i] += class_launches_[i];
            h.stats.class_bytes[i] += class_bytes_[i];
        }
        h.stats.iterations_run = iterations_;
        if (!c.ok()) return false;
        h.active_paths = paths_;
        return true;
    }

private:
    template <class Body>
    void capture(b2f_handle &h, Ctx &c, Body &body) {
        destroy();
        cudaStream_t cs = nullptr;
        c.check(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        if (!c.ok()) return;
        Ctx g = h.make_ctx(cs);
        b2f_stats scratch = h.stats;  // capture must not double-count launches
        scratch.iterations_run = 0;
        g.stats = &scratch;
        g.capturing = true;
        g.profiling = false;
        g.check(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
        if (g.ok()) body(g);
        cudaGraph_t graph = nullptr;
        g.check(cudaStreamEndCapture(cs, &graph));
        if (g.ok() && graph) g.check(cudaGraphInstantiate(&exec_, graph, 0));
        if (graph) cudaGraphDestroy(graph);
        cudaStreamDestroy(cs);
        launches_ = scratch.launches - h.stats.launches;
        for (int i = 0; i < B2F_MAX_KERNEL_CLASSES; ++i) {
            class_launches_[i] = scratch.class_launches[i] - h.stats.class_launches[i];
            class_bytes_[i] = scratch.class_bytes[i] - h.stats.class_bytes[i];
        }
        iterations_ = scratch.iterations_run;
        paths_ = h.active_paths;
        c.check(g.err);
        if (!c.ok()) destroy();
    }

    cudaGraphExec_t exec_ = nullptr;
    Key key_{};
    uint64_t launches_ = 0;
    uint64_t class_launches_[B2F_MAX_KERNEL_CLASSES] = {};
    double class_bytes_[B2F_MAX_KERNEL_CLASSES] = {};
    int iterations_ = 0;
    std::vector<double> paths_;
};

// ---------------------------------------------------------------------------------------------
// Shared kernels (pyramid.cu)
// ---------------------------------------------------------------------------------------------
// u8 / f32 image (arbitrary byte pitch) -> f32 plane * scale, two frames per launch.
void convert_pair(Ctx &c, int cls, const ImageView &a, const ImageView &b, Plane da, Plane db, float scale);
// cv::cuda::resize INTER_LINEAR semantics (top-left aligned; cudawarping/src/cuda/resize.cu:234-269),
// two planes per launch, result multiplied by `mul` (fuses cuda::multiply, tvl1flow.cpp:299-300).
void resize_linear_pair(Ctx &c, int cls, Plane sa, Plane sb, int srows, int scols, Plane da, Plane db,
                        int drows, int dcols, float inv_fx, float inv_fy, float mul);
void resize_linear_one(Ctx &c, int cls, Plane s, int srows, int scols, Plane d, int drows, int dcols,
                       float inv_fx, float inv_fy, float mul);
// planar (u, v) -> interleaved CV_32FC2 (cudaarithm split_merge.cu:99-148) and back (:239).
void merge_flow(Ctx &c, int cls, Plane u, Plane v, const ImageView &flow);
void split_flow(Ctx &c, int cls, const ImageView &flow, Plane u, Plane v);
void fill_plane(Ctx &c, Plane p, int rows, int cols, float value_bits_zero_only);
// cv::cuda::pyrDown f32 C1 (cudawarping/src/cuda/pyr_down.cu:55-173): 5x5 [1 4 6 4 1]/16, REFLECT101.
void pyr_down(Ctx &c, int cls, Plane s, int srows, int scols, Plane d, int drows, int dcols);
// same for an 8-bit pyramid held in float planes: the result is rounded like saturate_cast<uchar> (pyr_down.cu:172)
void pyr_down_u8(Ctx &c, int cls, Plane s, int srows, int scols, Plane d, int drows, int dcols);

// 2-D float32 TMA descriptor (128-byte CUtensorMap written to map_out); false when the driver entry point is missing.
bool tma_encode_2d_f32(void *map_out, const float *base, uint64_t width, uint64_t height, uint64_t pitch_bytes,
                       uint32_t box_w, uint32_t box_h);

// resize.cpp:76-84 scale rule: scale passed to the kernel is float(1/f).
static inline float inv_scale_from_sizes(int src, int dst) { return static_cast<float>(1.0 / (static_cast<double>(dst) / src)); }

// ---------------------------------------------------------------------------------------------
// Device helpers
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float sqrt_approx(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float rsqrt_approx(float x) {
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }
#endif

}  // namespace b2f
