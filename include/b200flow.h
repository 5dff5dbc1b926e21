/*
 * b200flow.h -- C ABI of libb200flow.so, the H100-native (sm_90a) dense optical-flow engine.
 *
 * This is the drop-in boundary for the cv::cuda::DenseOpticalFlow family of
 * opencv_contrib/modules/cudaoptflow.  Every entry point names the reference
 * interface it replaces (paths relative to opencv_contrib/modules/cudaoptflow).
 * Plain C: pointers + sizes only, no C++/torch types, no exceptions across the
 * boundary; every function returns a b2f_status.
 *
 * Images are described the way cv::cuda::GpuMat describes them
 * (opencv core cuda.hpp: data, step in BYTES, rows, cols, type flag), so the
 * C++ adapter (include/b200flow/cudaoptflow_compat.hpp) is a field-for-field copy.
 */
#ifndef B200FLOW_H_
#define B200FLOW_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define B2F_API
#else
#define B2F_API __attribute__((visibility("default")))
#endif

/* ---- status codes (reference: CV_Assert -> cv::Exception(StsAssert), cudaSafeCall ->
 *      cv::Exception(GpuApiCallError); include/b200flow/cudaoptflow_compat.hpp maps back) ---- */
typedef enum b2f_status {
    B2F_OK = 0,
    B2F_BAD_ARG = 1,          /* null pointer / invalid parameter value  (CV_Assert)          */
    B2F_UNSUPPORTED_TYPE = 2, /* image type not accepted by this algorithm (CV_Assert on type) */
    B2F_SIZE_MISMATCH = 3,    /* I0/I1/flow sizes differ                   (CV_Assert on size) */
    B2F_CUDA_ERROR = 4,       /* a CUDA runtime call failed; see b2f_last_cuda_error()          */
    B2F_NO_DEVICE = 5,        /* no usable sm_90 device                    (throw_no_cuda)      */
    B2F_OUT_OF_MEMORY = 6
} b2f_status;

/* ---- image type flags: numerically equal to OpenCV's CV_MAKETYPE values ---- */
enum {
    B2F_8UC1 = 0,   /* CV_8UC1  */
    B2F_32FC1 = 5,  /* CV_32FC1 */
    B2F_32FC2 = 13, /* CV_32FC2 */
    /* accepted by b2f_sparselk_calc only (the instantiations of cuda/pyrlk.cu's dispatcher table, src/pyrlk.cpp:195-203):
     * depth 8U / 16U / 32S / 32F with 1, 3 or 4 interleaved channels */
    B2F_16UC1 = 2, B2F_32SC1 = 4,
    B2F_8UC3 = 16, B2F_16UC3 = 18, B2F_32SC3 = 20, B2F_32FC3 = 21,
    B2F_8UC4 = 24, B2F_16UC4 = 26, B2F_32SC4 = 28, B2F_32FC4 = 29
};

/* Mirror of the GpuMat fields that cross the boundary (data/step/rows/cols/type). `data` is a
 * DEVICE pointer for b2f_calc and a HOST pointer for b2f_calc_host.  Rows may be pitched
 * (step >= cols*elemSize), i.e. ROIs of larger GpuMats are accepted. */
typedef struct b2f_image {
    void *data;
    size_t step; /* bytes */
    int rows;
    int cols;
    int type;
} b2f_image;

/* ---- parameter blocks; field order and defaults mirror the reference's create() ---- */

/* cv::cuda::OpticalFlowDual_TVL1::create  (include/opencv2/cudaoptflow.hpp:375-385) */
typedef struct b2f_tvl1_params {
    double tau;           /* 0.25 */
    double lambda;        /* 0.15 */
    double theta;         /* 0.3  */
    int nscales;          /* 5    */
    int warps;            /* 5    */
    double epsilon;       /* 0.01 */
    int iterations;       /* 300  */
    double scale_step;    /* 0.8  */
    double gamma;         /* 0.0  */
    int use_initial_flow; /* 0    */
} b2f_tvl1_params;

/* cv::cuda::FarnebackOpticalFlow::create  (cudaoptflow.hpp:285-293) */
typedef struct b2f_farneback_params {
    int num_levels;    /* 5   */
    double pyr_scale;  /* 0.5 */
    int fast_pyramids; /* 0   */
    int win_size;      /* 13  */
    int num_iters;     /* 10  */
    int poly_n;        /* 5   */
    double poly_sigma; /* 1.1 */
    int flags;         /* 0; B2F_OPTFLOW_* below */
} b2f_farneback_params;

enum {
    B2F_OPTFLOW_USE_INITIAL_FLOW = 4,    /* cv::OPTFLOW_USE_INITIAL_FLOW   */
    B2F_OPTFLOW_FARNEBACK_GAUSSIAN = 256 /* cv::OPTFLOW_FARNEBACK_GAUSSIAN */
};

/* cv::cuda::BroxOpticalFlow::create  (cudaoptflow.hpp:179-185) */
typedef struct b2f_brox_params {
    double alpha;          /* 0.197 flow smoothness              */
    double gamma;          /* 50.0  gradient constancy importance */
    double scale_factor;   /* 0.8   */
    int inner_iterations;  /* 5     */
    int outer_iterations;  /* 150   (cap on pyramid levels)       */
    int solver_iterations; /* 10    */
} b2f_brox_params;

/* cv::cuda::DensePyrLKOpticalFlow::create  (cudaoptflow.hpp:245-249) */
typedef struct b2f_denselk_params {
    int win_width;        /* 13 */
    int win_height;       /* 13 */
    int max_level;        /* 3  */
    int iters;            /* 30 */
    int use_initial_flow; /* 0  */
} b2f_denselk_params;

typedef struct b2f_handle b2f_handle;

/* ---- construction: replaces the static ::create() factories.  A NULL params pointer means
 *      "the reference's defaults".  Parameter validation happens in b2f_calc, exactly where the
 *      reference's CV_Asserts sit (src/tvl1flow.cpp:187-191, src/farneback.cpp:173-174,316-317,
 *      src/brox.cpp:134-135, src/pyrlk.cpp:240-243). ---- */
B2F_API void b2f_tvl1_default_params(b2f_tvl1_params *p);
B2F_API void b2f_farneback_default_params(b2f_farneback_params *p);
B2F_API void b2f_brox_default_params(b2f_brox_params *p);
B2F_API void b2f_denselk_default_params(b2f_denselk_params *p);

B2F_API int b2f_tvl1_create(const b2f_tvl1_params *p, b2f_handle **out);           /* src/tvl1flow.cpp:385-391 */
B2F_API int b2f_farneback_create(const b2f_farneback_params *p, b2f_handle **out); /* src/farneback.cpp:484-489 */
B2F_API int b2f_brox_create(const b2f_brox_params *p, b2f_handle **out);           /* src/brox.cpp:190-194 */
B2F_API int b2f_denselk_create(const b2f_denselk_params *p, b2f_handle **out);     /* src/pyrlk.cpp:402-405 */
B2F_API void b2f_destroy(b2f_handle *h);

/* ---- getters/setters: replace getTau()/setTau() ... (cudaoptflow.hpp:158-177,233-243,261-283,
 *      311-373).  Ids are per-algorithm; bools and ints travel as doubles. ---- */
typedef enum b2f_param_id {
    /* TV-L1 */
    B2F_TVL1_TAU = 100, B2F_TVL1_LAMBDA, B2F_TVL1_THETA, B2F_TVL1_NSCALES, B2F_TVL1_WARPS,
    B2F_TVL1_EPSILON, B2F_TVL1_ITERATIONS, B2F_TVL1_SCALE_STEP, B2F_TVL1_GAMMA,
    B2F_TVL1_USE_INITIAL_FLOW,
    /* TV-L1 knobs of the reference's CPU / OpenCL class (cv::optflow::DualTVL1OpticalFlow), set through b2f_set_param
     * only -- cv::cuda::OpticalFlowDual_TVL1::create has no such arguments:
     *   MEDIAN_FILTERING  1 = off (default), 3 or 5: cv::medianBlur of (u1, u2) before every block of MEDIAN_PERIOD
     *                     iterations (modules/optflow/src/tvl1flow.cpp:1377-1383);
     *   MEDIAN_PERIOD     iterations between two median passes = the CPU path's innerIterations (0 = once per warp);
     *                     CPU twin of (inner I, outer O, median k) = iterations I*O, MEDIAN_PERIOD I, MEDIAN_FILTERING k.
     *   INITIAL_FLOW_SOURCE  what useInitialFlow starts from: 0 = the caller's `flow` (default), 1 = this handle's own
     *                     previous result (zero on a fresh handle) -- the reference's CUDA class never reads the caller's
     *                     flow: it takes flowx / flowy from the buffer pool (src/tvl1flow.cpp:175-179,203-207), i.e.
     *                     whatever the previous call left there. */
    B2F_TVL1_MEDIAN_FILTERING = 120, B2F_TVL1_MEDIAN_PERIOD, B2F_TVL1_INITIAL_FLOW_SOURCE,
    /* Farneback */
    B2F_FARN_NUM_LEVELS = 200, B2F_FARN_PYR_SCALE, B2F_FARN_FAST_PYRAMIDS, B2F_FARN_WIN_SIZE,
    B2F_FARN_NUM_ITERS, B2F_FARN_POLY_N, B2F_FARN_POLY_SIGMA, B2F_FARN_FLAGS,
    /* Brox */
    B2F_BROX_ALPHA = 300, B2F_BROX_GAMMA, B2F_BROX_SCALE_FACTOR, B2F_BROX_INNER_ITERATIONS,
    B2F_BROX_OUTER_ITERATIONS, B2F_BROX_SOLVER_ITERATIONS,
    /* DensePyrLK */
    B2F_LK_WIN_WIDTH = 400, B2F_LK_WIN_HEIGHT, B2F_LK_MAX_LEVEL, B2F_LK_ITERS,
    B2F_LK_USE_INITIAL_FLOW,
    /* engine knobs (no reference counterpart) */
    B2F_ENGINE_FUSED_ITERS = 900, /* TV-L1: inner iterations fused per HBM pass (0 = auto)     */
    B2F_ENGINE_USE_GRAPH = 901,   /* capture the fixed schedule in a CUDA graph (default 1)    */
    B2F_ENGINE_KERNEL_PATH = 902, /* TV-L1: 0 = auto (persistent TMA kernel, centre tiles stored by TMA), 1 = unfused
                                     reference-shaped kernels, 2 = blocked kernel without TMA, 3 = TMA kernel without
                                     elect.sync, 4 = TMA loads with the STG epilogue, 5 = paired-strip TMA kernel
                                     (two pixels per thread row), 6 / 7 = 2x2 / 2x1-cluster kernels, 8 = two warp groups half an
                                     iteration apart, 9 = warps synchronise with their neighbours through mbarriers
                                     (11 = 9 with the TMA-store epilogue), 12 = row-skewed iterations behind
                                     split-phase mbarriers.  All bit-identical; 0 is the default.
                                     Brox: 0 = register-resident solver, one prepare + one solver launch per inner
                                     step, 1 = one launch per half sweep, 2 = shared-memory solver, 3 = all inner steps
                                     of a level in one cooperative launch.  All bit-identical.
                                     Farneback: 0 = auto (register-blocked quad kernel for winSize 13, the generic
                                     kernel otherwise), 1 = the generic kernel for every winSize, 2 = the
                                     register-blocked kernel with a per-pixel R1 gather, 3 = the persistent TMA
                                     kernel on levels with at least 2 x n_SM 64x64 tiles (0 elsewhere).  All agree to
                                     rounding; 3 is bit-identical to 0.  */
    B2F_ENGINE_AUX_PATH = 903,    /* variant of the secondary kernels.  TV-L1 warp: 0 = tiled kernel (I1 window of a
                                     64x32 tile staged in shared memory by TMA), 1 = tap-by-tap kernel (accumulation
                                     in the reference's order), 2 / 3 = separable kernel at 32 / 40 registers; 0, 2
                                     and 3 are bit-identical.  Farneback: fused iteration kernel
                                     at 0 = 128 registers (2 blocks / SM), 3 = 80, 4 = 64 registers, 5 = R1 gather
                                     with lanes on consecutive pixels, 6 = the simpler polynomial
                                     expansion and vertical-blur kernels.  All bit-identical.
                                     Brox (a test knob): 0 = the data term's reciprocal square root by rsqrtf, as the
                                     reference computes it (the default; up to 2 ulp, bits not specified by CUDA), 1 =
                                     correctly rounded (__frsqrt_rn), so that a float model can match the engine bit
                                     for bit.  Nothing else depends on it.                                             */
    /* Read-only: B2F_ENGINE_ACTIVE_PATH + s is what the last calc ran on pyramid level s (0 = full size); B2F_BAD_ARG
     * for a level the last calc did not solve.  TV-L1: an OR of b2f_tvl1_path flags.  A shape whose tensor maps cannot
     * be encoded falls back to the plain-load kernels; this says whether it did.  Farneback: the b2f_farneback_path of
     * the fused iteration kernel (0 with numIters = 0).  kernel_path 3 falls back to the fast kernel on levels with
     * fewer than 2 x n_SM 64x64 tiles or whose tensor maps cannot be encoded; this says whether it did.  Brox: the
     * b2f_brox_path of the solver in bits 0-7, and in bits 8-15 the solver iterations the first launch of each inner
     * step runs (all of them on a level that fits one 64x64 region or with B2F_BROX_PATH_COOP; the last launch of an
     * inner step runs the remainder; 0 for B2F_BROX_PATH_HALF_SWEEP, whose launch is half an iteration; at most 255).
     * kernel_path 3 falls back to kernel_path 0 on levels whose regions are not co-resident or that need more than one
     * solver launch per inner step; this says whether it did. */
    B2F_ENGINE_ACTIVE_PATH = 1000
} b2f_param_id;

/* Fused Farneback iteration kernels.  The box and gaussian windows share a value. */
typedef enum b2f_farneback_path {
    B2F_FARN_PATH_TMA = 1,             /* persistent kernel, M tiles staged by TMA (kernel_path 3)                  */
    B2F_FARN_PATH_QUAD = 2,            /* register-blocked, quad R1 gather, 256 threads, 128 registers (the gaussian
                                          window always runs this one)                                              */
    B2F_FARN_PATH_QUAD_WIDE = 3,       /* the same at 512 threads: box levels with at most n_SM 64x32 tiles          */
    B2F_FARN_PATH_QUAD_R80 = 4,        /* 256 threads at 80 registers (aux_path 3)                                   */
    B2F_FARN_PATH_QUAD_R64 = 5,        /* 256 threads at 64 registers (aux_path 4)                                   */
    B2F_FARN_PATH_QUAD_TRANSPOSED = 6, /* 256 threads, lanes on consecutive pixels in the R1 gather (aux_path 5)     */
    B2F_FARN_PATH_FAST = 7,            /* register-blocked, per-pixel R1 gather (kernel_path 2)                      */
    B2F_FARN_PATH_GENERIC = 8          /* k_farn_iter: any winSize other than 13, or kernel_path 1                   */
} b2f_farneback_path;

/* Brox solver kernels (B2F_ENGINE_ACTIVE_PATH, bits 0-7). */
typedef enum b2f_brox_path {
    B2F_BROX_PATH_REG = 1,        /* register-resident fused red-black SOR, one prepare + solver launches per inner step */
    B2F_BROX_PATH_SMEM = 2,       /* shared-memory fused red-black SOR (kernel_path 2)                                  */
    B2F_BROX_PATH_HALF_SWEEP = 3, /* one launch per red or black half sweep (kernel_path 1)                             */
    B2F_BROX_PATH_COOP = 4        /* all inner steps of the level in one cooperative launch (kernel_path 3)             */
} b2f_brox_path;

typedef enum b2f_tvl1_path {
    B2F_TVL1_PATH_ITER_TMA = 1,       /* inner iterations: a persistent TMA-staged blocked kernel (kernel_path 0, 3-12) */
    B2F_TVL1_PATH_ITER_BLOCKED = 2,   /* inner iterations: the blocked kernel with plain loads                          */
    B2F_TVL1_PATH_ITER_UNFUSED = 4,   /* inner iterations: the unfused estimate_u / estimate_dual pair                  */
    B2F_TVL1_PATH_WARP_TILED = 8,     /* warp: the tiled kernel, I1 window staged by TMA                                */
    B2F_TVL1_PATH_WARP_UNTILED = 16   /* warp: the separable or tap-by-tap kernel                                       */
} b2f_tvl1_path;

/* cv::medianBlur for CV_32FC1, ksize 3 or 5, replicated border, not in place: the primitive behind
 * B2F_TVL1_MEDIAN_FILTERING (the reference's CPU path calls cv::medianBlur, modules/optflow/src/tvl1flow.cpp:1381-1382;
 * cv::cuda has no float median filter).  Pitched device planes (step a multiple of 4 bytes). */
B2F_API int b2f_median_blur_32f(const b2f_image *src, b2f_image *dst, int ksize, void *cuda_stream);

B2F_API int b2f_set_param(b2f_handle *h, int id, double value);
B2F_API int b2f_get_param(const b2f_handle *h, int id, double *value);

/* cv::Algorithm::getDefaultName(): "DenseOpticalFlow.OpticalFlowDual_TVL1" etc.
 * (src/tvl1flow.cpp:122, src/farneback.cpp:132, src/brox.cpp:67, src/pyrlk.cpp:394). */
B2F_API const char *b2f_default_name(const b2f_handle *h);

/* ---- the hot call: replaces DenseOpticalFlow::calc(I0, I1, flow, stream)
 *      (cudaoptflow.hpp:80; impls src/tvl1flow.cpp:170, src/farneback.cpp:167, src/brox.cpp:129,
 *      src/pyrlk.cpp:379).
 *   I0, I1 : device images, equal size/type.  TV-L1: 8UC1 (0..255) or 32FC1 (0..1, scaled x255);
 *            Farneback: 8UC1 or 32FC1 (no scaling); Brox: 32FC1 in [0,1]; DensePyrLK: 8UC1.
 *   flow   : device image, 32FC2, same size, allocated by the caller (the C++ adapter does the
 *            GpuMat::create the reference does inside calc).  Read first only when the
 *            algorithm's use-initial-flow option is set.
 *   stream : a cudaStream_t (as void*).  All work is ordered after the caller's prior work on
 *            that stream and is complete in stream order on return; no host synchronisation
 *            happens inside the call unless stream == NULL (legacy default stream: the call
 *            ends with a device synchronise, as the reference's launchers do). ---- */
B2F_API int b2f_calc(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *flow,
                     void *cuda_stream);

/* Same contract with HOST buffers (pinned or pageable): uploads I0/I1, runs b2f_calc, downloads
 * flow, all on `stream`; returns after the download has completed.  This is what a caller holding
 * cv::Mat frames does with GpuMat::upload/download around calc (samples/optical_flow.cpp:170-238). */
B2F_API int b2f_calc_host(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *flow,
                          void *cuda_stream);

/* Bytes of device workspace the handle holds (after the first calc) or would allocate for a
 * rows x cols input of `type` (replaces brox.cpp:112-122 getBufSize / BufferPool sizing). */
B2F_API size_t b2f_workspace_bytes(b2f_handle *h, int rows, int cols, int type);

/* ---- diagnostics ---- */
B2F_API const char *b2f_status_string(int status);
B2F_API int b2f_last_cuda_error(const b2f_handle *h); /* cudaError_t of the last failure */
B2F_API const char *b2f_version(void);

/* Kernel launch accounting for bench.py ("gpu_launches") and the roofline line.  Classes are
 * per algorithm; class 0 is always the dominant inner-loop kernel. */
#define B2F_MAX_KERNEL_CLASSES 16
typedef struct b2f_stats {
    uint64_t calls;                                /* b2f_calc invocations                        */
    uint64_t launches;                             /* kernel launches issued (graph nodes count)  */
    uint64_t class_launches[B2F_MAX_KERNEL_CLASSES];
    double class_ms[B2F_MAX_KERNEL_CLASSES];       /* CUDA-event time, only while profiling is on */
    double class_bytes[B2F_MAX_KERNEL_CLASSES];    /* algorithmic bytes moved by those launches   */
    int levels;                                    /* pyramid levels used by the last calc        */
    int iterations_run;                            /* inner iterations executed by the last calc  */
} b2f_stats;
B2F_API int b2f_get_stats(b2f_handle *h, b2f_stats *out); /* synchronises the profiling events */
B2F_API int b2f_reset_stats(b2f_handle *h);
B2F_API const char *b2f_kernel_class_name(const b2f_handle *h, int cls);
/* When on, every kernel launch is bracketed by CUDA events on the launching stream (graphs are
 * bypassed) so per-class device time can be read back with b2f_get_stats. */
B2F_API int b2f_set_profiling(b2f_handle *h, int on);


/* =============================================================================================
 * Adjacent components (SURVEY.md section 8f): what sits directly either side of calc().
 * ============================================================================================= */

/* ---- planar output: same contract as b2f_calc but the flow is written as two 32FC1 planes.
 *      The reference's consumers call calc() and then cuda::split (superres/src/optical_flow.cpp:
 *      557-574, 816-835); this skips the merge + split round trip.  With the algorithm's
 *      use-initial-flow option the planes are read first. ---- */
B2F_API int b2f_calc_uv(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *u, b2f_image *v,
                        void *cuda_stream);

/* ---- cv::cuda::interpolateFrames (cudalegacy.hpp:229, src/interpolate_frames.cpp:54-111,
 *      src/cuda/NPP_staging.cu:1648-1790 nppiStInterpolateFrames, :1838-1905 forward splat).
 *   frame0, frame1, fu, fv, bu, bv : device 32FC1 images of one size AND one step (the reference
 *            asserts equal steps, interpolate_frames.cpp:82).
 *   pos    : time position in [0,1].
 *   new_frame : device 32FC1 output, same size/step.
 *   buf    : device 32FC1 scratch of 6*rows x cols, same step, laid out like the reference's
 *            (coverage0, coverage1, fwdU, fwdV, bwdU, bwdV); zeroed by the call.
 *   flags  : B2F_INTERP_REFERENCE reproduces the reference bit-for-bit in formula, including its
 *            three defects (the 4th splat lands in bwdU a second time so bwdV stays 0,
 *            NPP_staging.cu:1779-1787; both samples of the "visible in both" branch read frame0,
 *            :1666; the coverage clear indexes by width not stride, :1985-1996);
 *            B2F_INTERP_CORRECTED fixes the three.  Float atomics: the sum order is not fixed,
 *            results agree to rounding (as in the reference). ---- */
enum { B2F_INTERP_REFERENCE = 0, B2F_INTERP_CORRECTED = 1 };
B2F_API int b2f_interpolate_frames(const b2f_image *frame0, const b2f_image *frame1, const b2f_image *fu,
                                   const b2f_image *fv, const b2f_image *bu, const b2f_image *bv, float pos,
                                   b2f_image *new_frame, b2f_image *buf, int flags, void *cuda_stream);

/* ---- batched frame-pair front end for one GPU (SURVEY.md 8b / 8e): N engine handles on N streams, pairs dealt
 *      round robin -- the pattern of the reference's own multi-stream test (test/test_optflow.cpp:468-528).
 *      algo: 1 TV-L1, 2 Farneback, 3 Brox, 4 DensePyrLK; params: the matching b2f_*_params (NULL = defaults).
 *      Sharding over GPUs / processes and the NCCL result gather stay with the caller's process framework
 *      (opencv_contrib_b200/batch.py over torch.distributed). ---- */
typedef struct b2f_batch b2f_batch;
B2F_API int b2f_batch_create(int algo, const void *params, int n_streams, b2f_batch **out);
B2F_API int b2f_batch_streams(const b2f_batch *b);
B2F_API b2f_handle *b2f_batch_engine(b2f_batch *b, int i); /* borrowed: engine i, e.g. for b2f_get_stats */
B2F_API int b2f_batch_set_param(b2f_batch *b, int id, double value); /* every engine */
/* n_pairs device-resident pairs -> flows.  Forked from / joined to `stream` with events only: no host
 * synchronisation, CUDA events on `stream` bracket the whole batch. */
B2F_API int b2f_batch_run_device(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1,
                                 b2f_image *flow, void *cuda_stream);
/* n_pairs HOST pairs -> host flows: one worker thread per stream runs b2f_calc_host on its share, so the copies
 * of one pair overlap the solves of the others.  Returns when every flow has landed. */
B2F_API int b2f_batch_run_host(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1, b2f_image *flow);
/* ---- multi-GPU: one process per GPU, pairs sharded by the caller (rank r owns a contiguous block), NO data-path
 *      collective; the only exchange is the gather of the finished flows to rank `dst`, done here over NCCL
 *      (ncclSend / ncclRecv; libnccl.so.2 is taken from the process or dlopen'ed -- never a link dependency).
 *      Every flow is sent as soon as its own solve has finished, on a communication stream, so transfers overlap
 *      the remaining solves.  Replaces what callers of the reference do by hand after looping over calc().
 *        b2f_comm_unique_id   rank 0 creates the 128-byte NCCL id, the caller distributes it (any side channel)
 *        b2f_comm_create      collective over all ranks; binds to the CURRENT device; nranks == 1 needs no NCCL
 *        b2f_comm_adopt       wrap an ncclComm_t the application already owns (not destroyed by b2f_comm_destroy)
 *        b2f_batch_run_device_gather   like b2f_batch_run_device, plus the gather: on rank `dst`, gathered[r * n_pairs + i]
 *                             receives pair i of rank r (contiguous CV_32FC2, step == cols * 8; the entry for r == dst may
 *                             alias flow[i]); other ranks pass NULL.  Same n_pairs and sizes on every rank.
 *      Everything is ordered on `cuda_stream` like b2f_batch_run_device: no host synchronisation. ---- */
typedef struct b2f_comm b2f_comm;
B2F_API int b2f_comm_available(void);
B2F_API int b2f_comm_unique_id(void *id128, size_t bytes);
B2F_API int b2f_comm_create(const void *id128, size_t bytes, int rank, int nranks, b2f_comm **out);
B2F_API int b2f_comm_adopt(void *nccl_comm, b2f_comm **out);
B2F_API int b2f_comm_rank(const b2f_comm *c);
B2F_API int b2f_comm_nranks(const b2f_comm *c);
B2F_API int b2f_comm_last_nccl_error(const b2f_comm *c);
B2F_API void b2f_comm_destroy(b2f_comm *c);
B2F_API int b2f_batch_run_device_gather(b2f_batch *b, int n_pairs, const b2f_image *I0, const b2f_image *I1,
                                        b2f_image *flow, b2f_comm *comm, int dst, b2f_image *gathered, void *cuda_stream);

B2F_API uint64_t b2f_batch_launches(b2f_batch *b);
B2F_API int b2f_batch_reset_stats(b2f_batch *b);
B2F_API void b2f_batch_destroy(b2f_batch *b);

/* ---- video front end: consecutive frames of one stream -> flow(k-1 -> k).
 *      Each pushed HOST frame is uploaded once (the previous frame stays resident), the solve for
 *      pair k overlaps the upload of frame k+1 and the download of flow k-1 (three streams, events,
 *      no host synchronisation inside push), and with `warm_start` the previous pair's flow seeds
 *      the next solve (tvl1flow.cpp:203-207,249-256 useInitialFlow; farneback.cpp:179-188,398-404
 *      OPTFLOW_USE_INITIAL_FLOW; the temporal chaining the reference's test does by hand,
 *      test_optflow.cpp:328-334).  `depth` = pairs in flight (ring of host-visible results). ---- */
typedef struct b2f_video b2f_video;
B2F_API int b2f_video_create(b2f_handle *h, int rows, int cols, int type, int depth, int warm_start,
                             b2f_video **out);
/* Enqueue frame k (host pointer, `step` bytes per row; pinned memory makes the copy asynchronous).
 * For k >= 1 a solve for pair (k-1, k) is enqueued and *pair_index receives k-1; for k = 0 it
 * receives -1.  Blocks only when `depth` pairs are already in flight. */
B2F_API int b2f_video_push(b2f_video *v, const void *host_frame, size_t step, int64_t *pair_index);
/* Wait for pair `pair_index` and copy its 32FC2 flow to host memory (`step` bytes per row).
 * Pairs must be fetched before they fall `depth` behind the newest push. */
B2F_API int b2f_video_fetch(b2f_video *v, int64_t pair_index, void *host_flow, size_t step);
/* Zero-copy variant: waits for the pair and returns a pointer into the front end's pinned result ring
 * (rows of `*step` bytes).  The memory stays valid until `depth` further pairs have been pushed. */
B2F_API int b2f_video_fetch_view(b2f_video *v, int64_t pair_index, const float **host_flow, size_t *step);
B2F_API void b2f_video_destroy(b2f_video *v);

/* ---- cv::cuda::SparsePyrLKOpticalFlow (cudaoptflow.hpp:189-226; src/pyrlk.cpp:153-236,344-376;
 *      src/cuda/pyrlk.cu:148-345): pyramidal Lucas-Kanade for a list of points.  Images: device CV_8UC1 or
 *      CV_32FC1 (the reference additionally instantiates 16U / 32S and 3 / 4 channels: not built here).
 *      prev_pts / next_pts: device arrays of n_points interleaved (x, y) float32 -- the reference's 1 x N
 *      CV_32FC2 GpuMat; status: n_points bytes (1 = tracked); err: n_points float32 or NULL.  next_pts is
 *      read first only when use_initial_flow is set.  A point that leaves the image or whose 2x2 matrix is
 *      singular keeps the coordinates of the last level that updated it and gets status 0 on level 0,
 *      exactly as the reference kernel returns early (pyrlk.cu:162-168,232-238,256-262). ---- */
typedef struct b2f_sparselk_params {
    int win_width;        /* 21 */
    int win_height;       /* 21 */
    int max_level;        /* 3  */
    int iters;            /* 30 */
    int use_initial_flow; /* 0  */
} b2f_sparselk_params;
typedef struct b2f_sparse b2f_sparse;
B2F_API void b2f_sparselk_default_params(b2f_sparselk_params *p);
B2F_API int b2f_sparselk_create(const b2f_sparselk_params *p, b2f_sparse **out);
B2F_API int b2f_sparselk_set_params(b2f_sparse *h, const b2f_sparselk_params *p);
B2F_API int b2f_sparselk_get_params(const b2f_sparse *h, b2f_sparselk_params *p);
B2F_API int b2f_sparselk_calc(b2f_sparse *h, const b2f_image *prev_img, const b2f_image *next_img,
                              const float *prev_pts, float *next_pts, unsigned char *status, float *err,
                              int n_points, void *cuda_stream);
B2F_API void b2f_sparselk_destroy(b2f_sparse *h);

/* ---- Middlebury .flo files and the reference's error measures (host side).
 *      Format: float tag 202021.25 ("PIEH"), int32 width, int32 height, then rows of interleaved
 *      (u, v) float32 (optflow/test/test_tvl1optflow.cpp:49-108,
 *      optflow/samples/optical_flow_evaluation.cpp:23-71). ---- */
B2F_API int b2f_flo_read_size(const char *path, int *rows, int *cols);
B2F_API int b2f_flo_read(const char *path, float *flow, size_t step, int rows, int cols);
B2F_API int b2f_flo_write(const char *path, const float *flow, size_t step, int rows, int cols);

enum { B2F_ERR_ENDPOINT = 0, B2F_ERR_ANGULAR_REFERENCE = 1, B2F_ERR_ANGULAR = 2 };
/* Per-pixel error map between two HOST 32FC2 fields (NaN where either flow is invalid: NaN or
 * |component| >= 1e9, optical_flow_evaluation.cpp:23-26).  B2F_ERR_ANGULAR_REFERENCE keeps the
 * sample's operator precedence, acos(u1.u2 / |u1| * |u2|) (:67); B2F_ERR_ANGULAR is the intended
 * acos(u1.u2 / (|u1| |u2|)). */
B2F_API int b2f_flow_error_map(const float *flow1, size_t step1, const float *flow2, size_t step2, int rows,
                               int cols, int measure, float *err, size_t err_step);
typedef struct b2f_error_stats {
    double mean, stddev;   /* meanStdDev over the mask (:126-130)                          */
    double r[5];           /* fraction with error > {0.5, 1, 2, 5, 10} (:74-93,133-139)    */
    double a[3];           /* error value at the {0.5, 0.75, 0.95} quantiles from a        */
                           /* 1024-bin histogram over [0, max] (:94-105,141-163)           */
    double max;
    int64_t count;         /* masked pixels                                                */
} b2f_error_stats;
/* mask: optional HOST 8-bit mask (non-zero = use), NULL = all pixels.  A NaN error propagates through
 * mean/stddev as it does through cv::meanStdDev, compares false in the R statistics and lands in no
 * histogram bin. */
B2F_API int b2f_flow_error_stats(const float *err, size_t err_step, const unsigned char *mask, size_t mask_step,
                                 int rows, int cols, b2f_error_stats *out);
/* The reference's regression criterion (test_tvl1optflow.cpp:114-142): among gold pixels that are
 * valid, the fraction whose squared endpoint error is <= threshold^2; a test passes when it is
 * >= expected accuracy (0.95 at threshold 0.1). */
B2F_API int b2f_flow_accuracy(const float *gold, size_t gold_step, const float *flow, size_t flow_step, int rows,
                              int cols, double threshold, double *fraction);

#ifdef __cplusplus
}
#endif
#endif /* B200FLOW_H_ */
