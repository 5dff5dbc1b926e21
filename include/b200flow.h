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

/* cv::optflow::createOptFlow_DeepFlow (optflow.hpp; defaults of the OpticalFlowDeepFlow constructor,
 * modules/optflow/src/deepflow.cpp:62-73).  Inputs 8UC1 or 32FC1 of equal size and type, output 32FC2; the caller's
 * flow is never read (the reference discards it, deepflow.cpp:132,146), so the video front end's warm start is
 * refused.  sigma, downscale_factor, alpha, delta, gamma and omega are the reference's float members: the
 * engine rounds them to float.  The pre-smoothing kernel length floor(3 sigma) * 2 + 1 must be 3 (0 < sigma < 1).  The reference class
 * does not override getDefaultName; b2f_default_name reports "DenseOpticalFlow.DeepFlow". */
typedef struct b2f_deepflow_params {
    double sigma;               /* 0.6  Gaussian pre-smoothing                        */
    int min_size;               /* 25   stop the pyramid when a side is <= min_size   */
    double downscale_factor;    /* 0.95 */
    int fixed_point_iterations; /* 5    */
    int sor_iterations;         /* 25   */
    double alpha;               /* 1.0  smoothness (VariationalRefinement gets 4 alpha) */
    double delta;               /* 0.5  colour constancy (gets delta / 3)             */
    double gamma;               /* 5.0  gradient constancy (gets gamma / 3)           */
    double omega;               /* 1.6  SOR relaxation                                */
    int max_layers;             /* 200  levels below the source at most (buildPyramid's loop), so up to
                                           max_layers + 1 levels; 0 = the source level only */
} b2f_deepflow_params;

/* cv::DISOpticalFlow (opencv's video module, dense inverse search).  Inputs 8UC1 of equal size (anything else:
 * B2F_UNSUPPORTED_TYPE), output 32FC2.  With use_initial_flow the caller's 32FC2 flow is read as the initial flow
 * (cv::DISOpticalFlow::calc reads a flow of the frame's size and type): it is resized (INTER_LINEAR) to the coarsest
 * level times 1 / 2^coarsest, and there each patch starts from it or from zero flow, whichever has the lower SSD.  On a
 * single-level pyramid (finest == coarsest == 0) this is cv2's rule bit for bit; on deeper pyramids cv2's rule has not
 * been established and the engine's result differs from cv2's.  Without it the coarsest level starts from zero.  Spatial propagation follows OpenCV's OpenCL kernels (every
 * patch row scanned, then every patch descends), not its CPU path, so with propagation on the result agrees with
 * cv2.DISOpticalFlow statistically, not bit for bit.  Only patch_size 8 is built (all three presets use it); any other
 * size, a stride outside 1..patch_size, a finest_scale outside 0..5, or a frame too small for finest_scale is refused
 * with B2F_BAD_ARG.  The coarsest level is min(coarsest_scale, the automatic rule) (coarsest_scale -1: the automatic
 * rule).  The refinement stage is VariationalRefinement with omega 1.6 and 5 SOR iterations, as DIS configures it.
 * cv2 reports the default name "my_object" for this class; b2f_default_name reports the same. */
typedef struct b2f_dis_params {
    int finest_scale;                      /* 2 (MEDIUM: 1)                                    */
    int coarsest_scale;                    /* -1 = automatic                                   */
    int patch_size;                        /* 8                                                */
    int patch_stride;                      /* 4 (MEDIUM: 3)                                    */
    int grad_descent_iterations;           /* 16 (ULTRAFAST: 12, MEDIUM: 25)                   */
    int variational_refinement_iterations; /* 5 (ULTRAFAST: 0)                                 */
    double alpha;                          /* 20  refinement smoothness                        */
    double delta;                          /* 5   refinement colour constancy                  */
    double gamma;                          /* 10  refinement gradient constancy                */
    double epsilon;                        /* 0.01 refinement robust-function epsilon          */
    int use_mean_normalization;            /* 1 */
    int use_spatial_propagation;           /* 1 */
    int use_initial_flow;                  /* 0  read the caller's flow as the initial flow    */
} b2f_dis_params;

/* cv::DISOpticalFlow::PRESET_* */
enum { B2F_DIS_PRESET_ULTRAFAST = 0, B2F_DIS_PRESET_FAST = 1, B2F_DIS_PRESET_MEDIUM = 2 };

/* cv::cuda::FastOpticalFlowBM (modules/cudalegacy/include/opencv2/cudalegacy.hpp:202-211; src/bm_fast.cpp:62-88,
 * src/cuda/bm_fast.cu).  Dense integer block matching: for every pixel the offset (x, y) in
 * [-sr, search_window - 1 - sr]^2, sr = search_window / 2, whose block_window x block_window sum of absolute differences
 * between I0 and I1 is least; both frames are extended with cudev's reflect-101 rule (one fold and a modulo, not the
 * CPU's iterative borderInterpolate).  Ties go to the least (k mod 128, k div 128) for k = y * search_window + x, as the
 * reference's 128-thread scan and reduction decide them.  Inputs 8UC1 of equal size (anything else:
 * B2F_UNSUPPORTED_TYPE), output 32FC2 (b2f_calc) or two 32FC1 planes (b2f_calc_uv, how the reference returns it); the
 * caller's flow is never read, so the video front end runs it without warm start.  Refused with B2F_BAD_ARG:
 *   search_window outside 1..109: the reference's kernel needs 4 * search_window^2 bytes of dynamic plus 1024 bytes of
 *       static shared memory without opting in to more than 48 KB, so 109 is its largest working size;
 *   an even block_window: the reference's column ring then overruns into the next CTA's buffer rows (a race);
 *   block_window above 31: this engine's warp keeps 32 - (block_window - 1) output columns (the reference has no limit).
 * The reference class is not a cv::Algorithm; b2f_default_name reports "DenseOpticalFlow.FastOpticalFlowBM".
 * B2F_ENGINE_ACTIVE_PATH + 0 after a calc: bits 0-7 the output columns per warp, bits 8-15 the tile rows, bit 16 set
 * when the (SAD, rank) key was compared in 64 bits (the window pair could overflow 32). */
typedef struct b2f_fastbm_params {
    int search_window; /* 21 */
    int block_window;  /* 7  */
} b2f_fastbm_params;

/* cv::VariationalRefinement (opencv's video module, cv2.VariationalRefinement_create): the caller's flow refined in
 * place by one calcUV call -- colour-constancy, gradient-constancy and smoothness terms, fixed-point steps of red-black
 * SOR; the solver DeepFlow runs per level and DIS runs as its refinement stage.  Inputs 8UC1 or 32FC1 of one type and
 * size (anything else: B2F_UNSUPPORTED_TYPE), converted to float without scaling; `flow` 32FC2 of the frame's size
 * (b2f_calc) or two 32FC1 planes (b2f_calc_uv) is always read first and receives the result.  Every parameter value is
 * accepted, as cv2 accepts it: an iteration count below one runs no step (the flow comes back unchanged); with
 * epsilon 0 cv2's output turns non-finite and this engine's need not.  A flow of another type is B2F_UNSUPPORTED_TYPE,
 * frames or a flow of another size B2F_SIZE_MISMATCH.  alpha, delta, gamma, epsilon and omega are the reference's float
 * members: the engine rounds them to float.  The video front end refuses this engine (it has no caller flow to
 * refine).  cv2 reports the default name "my_object"; b2f_default_name reports the same. */
typedef struct b2f_varref_params {
    int fixed_point_iterations; /* 5     outer (warping) iterations      */
    int sor_iterations;         /* 5     SOR iterations per outer step   */
    double omega;               /* 1.6   SOR relaxation                  */
    double alpha;               /* 20    smoothness                      */
    double delta;               /* 5     colour constancy                */
    double gamma;               /* 10    gradient constancy              */
    double epsilon;             /* 0.001 robust-function epsilon         */
} b2f_varref_params;

/* cv::calcOpticalFlowFarneback / cv::FarnebackOpticalFlow (opencv's video module, modules/video/src/optflowgf.cpp), bit
 * for bit equal to cv2 4.x's portable CPU path (cv2.setUseOptimized(False) with IPP off, the SSE baseline code every
 * x86-64 host runs; DESIGN §4.14).  Created by b2f_optflowgf_create from a b2f_farneback_params, whose fields are the
 * video class's create() arguments, and driven by the B2F_FARN_* parameter ids.  Unlike b2f_farneback_create (the
 * cv::cuda class) it follows the CPU class: centre-aligned level images blurred from the full-size frame, double box
 * sums, fastPyramids accepted and ignored.  Frames 8UC1 or 32FC1 of one type and size (cv2 also takes other depths:
 * here they are B2F_UNSUPPORTED_TYPE); the flow 32FC2 (b2f_calc) or two 32FC1 planes (b2f_calc_uv), read first with
 * B2F_OPTFLOW_USE_INITIAL_FLOW.  B2F_BAD_ARG: pyr_scale >= 1 (cv2 asserts), poly_n outside 1..B2F_OPTFLOWGF_MAX_POLY_N,
 * win_size outside 1..B2F_OPTFLOWGF_MAX_WIN_SIZE, or a deepest-level blur wider than 255 taps.  That blur has
 * ksize = max(cvRound(2.5 (1/scale - 1)) | 1, 3) at the deepest level's scale, so it is refused once 1/scale reaches about
 * 103: at pyr_scale 0.5 with num_levels >= 7 and a shorter side of at least 4096 (1/scale 128, ksize 319); never with the
 * default 5 levels.  A handle may be called on several streams: a call on another stream than the previous call waits
 * for it, since both use the handle's workspace.  b2f_default_name reports "DenseOpticalFlow.FarnebackOpticalFlow", as
 * cv2 does. */
enum { B2F_OPTFLOWGF_MAX_POLY_N = 15, B2F_OPTFLOWGF_MAX_WIN_SIZE = 255 };
/* B2F_ENGINE_ACTIVE_PATH + level (finest first) of an optflowgf handle: the window the level ran, plus AREA_LEVEL when
 * its images came through OpenCV's exact-half fast INTER_AREA rule */
enum { B2F_OPTFLOWGF_PATH_BOX = 1, B2F_OPTFLOWGF_PATH_GAUSSIAN = 2, B2F_OPTFLOWGF_PATH_AREA_LEVEL = 4 };

typedef struct b2f_handle b2f_handle;

/* ---- construction: replaces the static ::create() factories.  A NULL params pointer means
 *      "the reference's defaults".  Parameter validation happens in b2f_calc, exactly where the
 *      reference's CV_Asserts sit (src/tvl1flow.cpp:187-191, src/farneback.cpp:173-174,316-317,
 *      src/brox.cpp:134-135, src/pyrlk.cpp:240-243). ---- */
B2F_API void b2f_tvl1_default_params(b2f_tvl1_params *p);
B2F_API void b2f_farneback_default_params(b2f_farneback_params *p);
B2F_API void b2f_brox_default_params(b2f_brox_params *p);
B2F_API void b2f_denselk_default_params(b2f_denselk_params *p);
B2F_API void b2f_deepflow_default_params(b2f_deepflow_params *p);
B2F_API void b2f_dis_default_params(b2f_dis_params *p, int preset); /* DISOpticalFlow::create(preset) */
B2F_API void b2f_fastbm_default_params(b2f_fastbm_params *p);
B2F_API void b2f_varref_default_params(b2f_varref_params *p);

B2F_API int b2f_tvl1_create(const b2f_tvl1_params *p, b2f_handle **out);           /* src/tvl1flow.cpp:385-391 */
B2F_API int b2f_farneback_create(const b2f_farneback_params *p, b2f_handle **out); /* src/farneback.cpp:484-489 */
B2F_API int b2f_brox_create(const b2f_brox_params *p, b2f_handle **out);           /* src/brox.cpp:190-194 */
B2F_API int b2f_denselk_create(const b2f_denselk_params *p, b2f_handle **out);     /* src/pyrlk.cpp:402-405 */
B2F_API int b2f_deepflow_create(const b2f_deepflow_params *p, b2f_handle **out);   /* optflow deepflow.cpp:171-174 */
B2F_API int b2f_dis_create(const b2f_dis_params *p, b2f_handle **out);             /* NULL: the FAST preset */
B2F_API int b2f_fastbm_create(const b2f_fastbm_params *p, b2f_handle **out);       /* cudalegacy.hpp:202-211 */
B2F_API int b2f_varref_create(const b2f_varref_params *p, b2f_handle **out);       /* VariationalRefinement::create */
B2F_API int b2f_optflowgf_create(const b2f_farneback_params *p, b2f_handle **out); /* video FarnebackOpticalFlow */
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
    /* DeepFlow */
    B2F_DEEP_SIGMA = 500, B2F_DEEP_MIN_SIZE, B2F_DEEP_DOWNSCALE_FACTOR, B2F_DEEP_FIXED_POINT_ITERATIONS,
    B2F_DEEP_SOR_ITERATIONS, B2F_DEEP_ALPHA, B2F_DEEP_DELTA, B2F_DEEP_GAMMA, B2F_DEEP_OMEGA, B2F_DEEP_MAX_LAYERS,
    /* DIS */
    B2F_DIS_FINEST_SCALE = 600, B2F_DIS_COARSEST_SCALE, B2F_DIS_PATCH_SIZE, B2F_DIS_PATCH_STRIDE,
    B2F_DIS_GRADIENT_DESCENT_ITERATIONS, B2F_DIS_VARIATIONAL_REFINEMENT_ITERATIONS, B2F_DIS_VARIATIONAL_REFINEMENT_ALPHA,
    B2F_DIS_VARIATIONAL_REFINEMENT_DELTA, B2F_DIS_VARIATIONAL_REFINEMENT_GAMMA, B2F_DIS_VARIATIONAL_REFINEMENT_EPSILON,
    B2F_DIS_USE_MEAN_NORMALIZATION, B2F_DIS_USE_SPATIAL_PROPAGATION, B2F_DIS_USE_INITIAL_FLOW,
    /* FastOpticalFlowBM */
    B2F_FBM_SEARCH_WINDOW = 700, B2F_FBM_BLOCK_WINDOW,
    /* VariationalRefinement: a block of its own below the active-path ids, which start at 1000 */
    B2F_VR_FIXED_POINT_ITERATIONS = 950, B2F_VR_SOR_ITERATIONS, B2F_VR_OMEGA, B2F_VR_ALPHA, B2F_VR_DELTA, B2F_VR_GAMMA,
    B2F_VR_EPSILON,
    /* engine knobs (no reference counterpart) */
    B2F_ENGINE_FUSED_ITERS = 900, /* TV-L1: inner iterations fused per HBM pass (0 = auto)     */
    B2F_ENGINE_USE_GRAPH = 901,   /* capture the fixed schedule in a CUDA graph (default 1)    */
    B2F_ENGINE_KERNEL_PATH = 902, /* TV-L1: 0 = auto (persistent TMA kernel, centre tiles stored by TMA), 1 = unfused
                                     reference-shaped kernels, 2 = blocked kernel without TMA; any other value runs
                                     0.  All bit-identical.
                                     Brox: 0 = register-resident solver, one prepare + one solver launch per inner
                                     step, 1 = one launch per half sweep, 2 = shared-memory solver, 3 = all inner steps
                                     of a level in one cooperative launch.  All bit-identical.
                                     Farneback: 0 = auto (register-blocked quad kernel for winSize 13, the generic
                                     kernel otherwise), 1 = the generic kernel for every winSize, 2 = the
                                     register-blocked kernel with a per-pixel R1 gather, 3 = the persistent TMA
                                     kernel on levels with at least 2 x n_SM 64x64 tiles (0 elsewhere).  All agree to
                                     rounding; 3 is bit-identical to 0.  */
    B2F_ENGINE_AUX_PATH = 903,    /* variant of the secondary kernels.  TV-L1 warp: 0 = tiled kernel (I1 window of a
                                     64x32 tile staged in shared memory by TMA), 3 = separable kernel on every level;
                                     any other value runs 0.  Bit-identical.  Farneback: fused iteration kernel
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
     * solver launch per inner step; this says whether it did.  DeepFlow: the SOR iterations each solver launch of the
     * level runs (chosen from the level's shape; all of them on a level that fits one 64x64 region, which runs its
     * fixed-point steps in one launch).  DIS (s = pyramid scale, finest_scale .. coarsest): bits 0-7 the refinement's SOR
     * iterations per solver launch (0 without refinement), bits 8-23 the patch rows hs, bits 24-39 the patch columns ws.
     * VariationalRefinement (s = 0 only): the SOR iterations each solver launch runs, as DeepFlow's; 0 when the call runs
     * no SOR iteration. */
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
    B2F_TVL1_PATH_ITER_TMA = 1,       /* inner iterations: the persistent TMA-staged blocked kernel                      */
    B2F_TVL1_PATH_ITER_BLOCKED = 2,   /* inner iterations: the blocked kernel with plain loads                          */
    B2F_TVL1_PATH_ITER_UNFUSED = 4,   /* inner iterations: the unfused estimate_u / estimate_dual pair                  */
    B2F_TVL1_PATH_WARP_TILED = 8,     /* warp: the tiled kernel, I1 window staged by TMA                                */
    B2F_TVL1_PATH_WARP_UNTILED = 16   /* warp: the separable kernel                                                     */
} b2f_tvl1_path;

/* cv::medianBlur for CV_32FC1, ksize 3 or 5, replicated border, not in place: the primitive behind
 * B2F_TVL1_MEDIAN_FILTERING (the reference's CPU path calls cv::medianBlur, modules/optflow/src/tvl1flow.cpp:1381-1382;
 * cv::cuda has no float median filter).  Pitched device planes (step a multiple of 4 bytes). */
B2F_API int b2f_median_blur_32f(const b2f_image *src, b2f_image *dst, int ksize, void *cuda_stream);

/* Test support: out[i] = op(in[i]) for n device floats, through the very approximations the kernels use
 * (op 0: rcp.approx.ftz.f32, op 1: sqrt.approx.ftz.f32; one MUFU instruction each on sm_90a), so that a test can
 * tabulate them and check a model of them on every input.  NULL stream: synchronous. */
B2F_API int b2f_approx_probe(int op, const float *in, float *out, size_t n, void *cuda_stream);

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
 *            (coverage0, coverage1, fwdU, fwdV, bwdU, bwdV); the 6*rows x cols view is zeroed by the
 *            call, the columns past cols of a pitched buf are not touched.
 *   flags  : B2F_INTERP_REFERENCE reproduces the reference bit-for-bit in formula, including its
 *            three defects (the 4th splat lands in bwdU a second time so bwdV stays 0,
 *            NPP_staging.cu:1779-1787; both samples of the "visible in both" branch read frame0,
 *            :1666; the coverage clear indexes by width not stride, :1985-1996);
 *            B2F_INTERP_CORRECTED fixes the three.  Float atomics: the sum order of the six scratch
 *            accumulators is not fixed, so they agree to rounding (as in the reference); the output is a
 *            deterministic function of what the call leaves in buf. ---- */
enum { B2F_INTERP_REFERENCE = 0, B2F_INTERP_CORRECTED = 1 };
B2F_API int b2f_interpolate_frames(const b2f_image *frame0, const b2f_image *frame1, const b2f_image *fu,
                                   const b2f_image *fv, const b2f_image *bu, const b2f_image *bv, float pos,
                                   b2f_image *new_frame, b2f_image *buf, int flags, void *cuda_stream);

/* ---- cv::cuda::calcOpticalFlowBM (cudalegacy.hpp:196-200; src/bm.cpp:60-202, src/cuda/bm.cu:56-160): one vector
 *      per grid cell.  velSize = ((cols - bw + sw) / sw, (rows - bh + sh) / sh) for block (bw, bh) and shift (sw, sh);
 *      cell (i, j) compares the block at (j sw, i sh) of `curr` with `prev` at the candidate offsets (the reference's
 *      cmpBlocks receives its frames swapped: if curr is prev shifted by +s, the result is -s, kept for drop-in
 *      parity).  Candidates follow the reference's spiral over [-max_range, max_range]^2 minus the origin, relative to the
 *      start offset (the rounded previous velocity with use_previous, else 0); a candidate whose SAD is below
 *      2 bw bh is taken at once, ties with the best SAD are averaged, and a best above 128 bw bh falls back to the
 *      start offset.  The spiral is computed on the device, so no table buffer is needed.
 *   prev, curr : device 8UC1 of one size (else B2F_UNSUPPORTED_TYPE / B2F_SIZE_MISMATCH).
 *   velx, vely : device 32FC1 of velSize (else B2F_SIZE_MISMATCH), read first when use_previous is set.
 *   B2F_BAD_ARG: a block or shift side below 1, a range below 0 or above B2F_BM_MAX_RANGE, 128 bw bh above INT_MAX (the
 *      reference's escape level overflows), or an empty velSize.
 *   Asynchronous on `stream` like b2f_calc (a NULL stream ends with a device synchronise). ---- */
enum { B2F_BM_MAX_RANGE = 16383 };
B2F_API int b2f_calc_optical_flow_bm_size(int rows, int cols, int block_width, int block_height, int shift_width,
                                          int shift_height, int max_range_width, int max_range_height, int *vel_rows,
                                          int *vel_cols, int *table_len);
B2F_API int b2f_calc_optical_flow_bm(const b2f_image *prev, const b2f_image *curr, int block_width, int block_height,
                                     int shift_width, int shift_height, int max_range_width, int max_range_height,
                                     int use_previous, b2f_image *velx, b2f_image *vely, void *cuda_stream);

/* ---- batched frame-pair front end for one GPU (SURVEY.md 8b / 8e): N engine handles on N streams, pairs dealt
 *      round robin -- the pattern of the reference's own multi-stream test (test/test_optflow.cpp:468-528).
 *      algo: 1 TV-L1, 2 Farneback, 3 Brox, 4 DensePyrLK, 5 DeepFlow, 6 DIS, 7 FastOpticalFlowBM, 8 VariationalRefinement
 *      (each pair's flow is read and refined in place), 9 the video module's Farneback (b2f_optflowgf_create; params a
 *      b2f_farneback_params); params: the matching b2f_*_params (NULL = defaults).
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
 *      test_optflow.cpp:328-334).  `depth` = pairs in flight (ring of host-visible results).  A
 *      VariationalRefinement handle is refused with B2F_BAD_ARG: it refines a caller's flow, which the frame loop does
 *      not have, and the loop reuses its flow slots. ---- */
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

/* ---- superres: cv::superres::createSuperResolution_BTVL1_CUDA (modules/superres/src/btv_l1_cuda.cpp, src/cuda/
 *      btv_l1_gpu.cu): bilateral total-variation L1 multi-frame super-resolution of a video, on the optical flows of one of
 *      the engines above (TV-L1, Farneback, Brox or DensePyrLK through b2f_calc_ext's conversion) or of flows the caller
 *      supplies.  Frames are device 8UC1, 8UC3 or 8UC4 (anything else: B2F_UNSUPPORTED_TYPE) of one size per stream
 *      (else B2F_SIZE_MISMATCH).  The reference's pull schedule (nextFrame reads 2R + 1 frames first, then one per output)
 *      runs in the library: while b2f_superres_wants_frame says so, push the next frame (NULL = end of stream); then
 *      b2f_superres_pop returns the next output, rows*scale - 2 btv_kernel_size by cols*scale - 2 btv_kernel_size, as
 *      8UC{1,3,4} (the reference's nextFrame) or 32FC{1,3,4} (the float estimate before convertTo), until it reports no
 *      output at the end.  N frames give N outputs.  scale and temporal_area_radius are read when a stream's first frame
 *      arrives; the other parameters each time a frame is processed.  Every reference CV_Assert (btv_l1_cuda.cpp:310-316)
 *      plus an even or > 31 blur size, a radius above B2F_SR_MAX_RADIUS or an output of no pixels returns B2F_BAD_ARG
 *      from the push or pop that would process.  All work is on `cuda_stream`, without host synchronisation
 *      (a NULL stream ends each call with a device synchronise). ---- */
typedef struct b2f_superres_params {
    int scale;                /* 4    */
    int iterations;           /* 180  */
    double tau;               /* 1.3  */
    double lambda;            /* 0.03 */
    double alpha;             /* 0.7  */
    int btv_kernel_size;      /* 7    */
    int blur_kernel_size;     /* 5    */
    double blur_sigma;        /* 0.0  */
    int temporal_area_radius; /* 4    */
} b2f_superres_params;
enum { B2F_SR_MAX_RADIUS = 15 };
enum {
    B2F_SR_SCALE = 800, B2F_SR_ITERATIONS, B2F_SR_TAU, B2F_SR_LAMBDA, B2F_SR_ALPHA, B2F_SR_BTV_KERNEL_SIZE,
    B2F_SR_BLUR_KERNEL_SIZE, B2F_SR_BLUR_SIGMA, B2F_SR_TEMPORAL_AREA_RADIUS
};
typedef struct b2f_superres b2f_superres;
B2F_API void b2f_superres_default_params(b2f_superres_params *p);
/* flow: a TV-L1, Farneback, Brox or DensePyrLK handle (borrowed, else B2F_BAD_ARG), or NULL: the caller pushes flows */
B2F_API int b2f_superres_create(const b2f_superres_params *p, b2f_handle *flow, b2f_superres **out);
B2F_API int b2f_superres_set_flow(b2f_superres *sr, b2f_handle *flow);
B2F_API int b2f_superres_set_param(b2f_superres *sr, int id, double value); /* also B2F_ENGINE_USE_GRAPH */
B2F_API int b2f_superres_get_param(const b2f_superres *sr, int id, double *value);
B2F_API int b2f_superres_wants_frame(const b2f_superres *sr, int *wants);
/* readNextFrame: with a flow engine; frame NULL = end of stream */
B2F_API int b2f_superres_push(b2f_superres *sr, const b2f_image *frame, void *cuda_stream);
/* without one: the frame with 32FC1 flows previous -> frame (fwd) and frame -> previous (bwd); ignored for the first */
B2F_API int b2f_superres_push_flows(b2f_superres *sr, const b2f_image *frame, const b2f_image *fwd_u,
                                    const b2f_image *fwd_v, const b2f_image *bwd_u, const b2f_image *bwd_v,
                                    void *cuda_stream);
/* *produced = 1 when `out` received the next output, 0 at the end of the stream */
B2F_API int b2f_superres_pop(b2f_superres *sr, b2f_image *out, int *produced, void *cuda_stream);
B2F_API int b2f_superres_output_size(const b2f_superres *sr, int *rows, int *cols); /* after the first frame */
B2F_API int b2f_superres_reset(b2f_superres *sr);           /* a new stream */
B2F_API int b2f_superres_collect_garbage(b2f_superres *sr); /* a new stream, device memory released */
B2F_API int b2f_superres_get_stats(b2f_superres *sr, b2f_stats *out);
B2F_API int b2f_superres_reset_stats(b2f_superres *sr);
B2F_API int b2f_superres_last_cuda_error(const b2f_superres *sr);
B2F_API void b2f_superres_destroy(b2f_superres *sr);
/* superres's GpuOpticalFlow::calc (superres/src/optical_flow.cpp:456-497): 8UC{1,3,4} frames of one type and size are
 * converted to the engine's work type (cudev's 15-bit BGR(A)->gray rule, then x float(1/255) for Brox's 32FC1, 8UC1 for
 * the others), then flow1 = interleaved 32FC2, or with flow2 planar u / v 32FC1.  TV-L1, Farneback, Brox, DensePyrLK. */
B2F_API int b2f_calc_ext(b2f_handle *h, const b2f_image *I0, const b2f_image *I1, b2f_image *flow1, b2f_image *flow2,
                         void *cuda_stream);

/* ---- cudaimgproc corners: cv::cuda::CornernessCriteria and cv::cuda::CornersDetector (modules/cudaimgproc/include/
 *      opencv2/cudaimgproc.hpp:538-620; src/corners.cpp, src/gftt.cpp, src/cuda/corners.cu, src/cuda/gftt.cu).
 *   Response (b2f_harris_create / b2f_mineig_create + b2f_corners_compute): src device 8UC1 or 32FC1 (else
 *      B2F_UNSUPPORTED_TYPE), pitched or an ROI; dst device 32FC1 of the same size.  The derivatives are the reference's
 *      Sobel (ksize 1, 3, 5, 7) or Scharr (ksize <= 0) filters with scale 1 / (2^(ksize' - 1) blockSize (2 if ksize < 0)
 *      (255 for 8U)) folded into the smoothing kernel, then the blockSize x blockSize sums of dx^2, dx dy, dy^2 read the
 *      derivatives through the border rule again.  Harris: a c - b^2 - k (a + c)^2; min-eigenvalue: with a, c halved,
 *      (a + c) - sqrt((a - c)^2 + b^2).  border_type: 4 BORDER_REFLECT101, 1 BORDER_REPLICATE or 2 BORDER_REFLECT, with
 *      cudev's rules (one fold and a modulo).  One fused kernel: no intermediate planes; asynchronous on `cuda_stream`
 *      (a NULL stream ends with a device synchronise).  B2F_BAD_ARG: another border or ksize, a blockSize outside 1..31
 *      (departure: the reference accepts any; 31 keeps the block-sum halo inside one 32 x 16 tile).
 *   GoodFeaturesToTrack (b2f_gftt_*): the reference's preconditions (qualityLevel > 0, minDistance >= 0, maxCorners >= 0;
 *      B2F_BAD_ARG at creation), criterion aperture 3 and BORDER_REFLECT101.  b2f_gftt_detect writes up to `capacity`
 *      (x, y) float pairs to corners_dev -- integer positions, strongest first, the reference's 1 x N CV_32FC2 -- and N
 *      to *count_dev (device memory).  capacity must be at least b2f_gftt_capacity.  Departures from the reference:
 *        - no host synchronisation: the maximum response is folded on the device, candidates are counted, sorted and
 *          selected on the device; the call is asynchronous and can be captured in a CUDA graph.  The one exception:
 *          the first detect on a new image size synchronises the stream before it re-lays out the handle's workspace;
 *          inside a capture that call is refused (B2F_BAD_ARG), so run one detect of that size first;
 *        - candidates of equal response are ordered by raster index, higher first (CPU cv::goodFeaturesToTrack's
 *          tie order); the reference's unstable sort leaves it unspecified;
 *        - when there are more than max(1000, int(0.05 rows cols)) candidates, the first that many in this order are
 *          kept (the reference keeps whichever its atomics appended first);
 *        - the maximum that qualityLevel scales ignores the mask, as in the CUDA reference (gftt.cpp:120); CPU
 *          cv::goodFeaturesToTrack takes it under the mask.
 *      With minDistance >= 1 the result equals the reference's sequential grid rule (gftt.cpp:147-206) exactly, cell
 *      cvRound(minDistance) included; it is computed as greedy selection in priority order, in parallel rounds. ---- */
typedef struct b2f_corners b2f_corners;
B2F_API int b2f_harris_create(int src_type, int block_size, int ksize, double k, int border_type,
                              b2f_corners **out);                                                  /* corners.cpp:179-182 */
B2F_API int b2f_mineig_create(int src_type, int block_size, int ksize, int border_type, b2f_corners **out); /* :184-187 */
/* CornernessCriteria::compute (cudaimgproc.hpp:566) */
B2F_API int b2f_corners_compute(b2f_corners *h, const b2f_image *src, b2f_image *dst, void *cuda_stream);
typedef struct b2f_gftt_params {
    int max_corners;      /* 1000 (0: no limit) */
    double quality_level; /* 0.01 */
    double min_distance;  /* 0.0  */
    int block_size;       /* 3    */
    int use_harris;       /* 0    */
    double harris_k;      /* 0.04 */
} b2f_gftt_params;
B2F_API void b2f_gftt_default_params(b2f_gftt_params *p);
/* createGoodFeaturesToTrackDetector (cudaimgproc.hpp:610-620, gftt.cpp:217-222); NULL params: the defaults */
B2F_API int b2f_gftt_create(int src_type, const b2f_gftt_params *p, b2f_corners **out);
/* setMaxCorners / setMinDistance (cudaimgproc.hpp:596-599) and the other create() arguments */
B2F_API int b2f_gftt_set_params(b2f_corners *h, const b2f_gftt_params *p);
B2F_API int b2f_gftt_get_params(const b2f_corners *h, b2f_gftt_params *p);
/* the largest N a detect on a rows x cols image can return: min(maxCorners, max(1000, int(0.05 rows cols))) */
B2F_API int b2f_gftt_capacity(const b2f_corners *h, int rows, int cols, int *capacity);
/* CornersDetector::detect (cudaimgproc.hpp:589, gftt.cpp:107-214); mask: device 8UC1 of the image size or NULL */
B2F_API int b2f_gftt_detect(b2f_corners *h, const b2f_image *image, const b2f_image *mask, float *corners_dev,
                            int capacity, int *count_dev, void *cuda_stream);
/* What the last detect did (no reference counterpart): candidates found, candidates kept after the capacity cut, whether
 * the cut applied, and the rounds of the minDistance selection (0 with minDistance < 1).  Waits for `cuda_stream`. */
typedef struct b2f_gftt_info {
    int candidates;
    int kept;
    int capped;
    int rounds;
} b2f_gftt_info;
B2F_API int b2f_gftt_last_info(b2f_corners *h, b2f_gftt_info *out, void *cuda_stream);
B2F_API int b2f_corners_last_cuda_error(const b2f_corners *h);
B2F_API void b2f_corners_destroy(b2f_corners *h);

/* ---- the video module's pyramidal Lucas-Kanade tracker: cv::buildOpticalFlowPyramid, cv::calcOpticalFlowPyrLK and
 *      cv::SparsePyrLKOpticalFlow (video/tracking.hpp), bit for bit equal to cv2 4.13's x86 build, including the order in
 *      which it adds its float sums (DESIGN §4.13).  This is a second tracker next to b2f_sparselk_* (cv::cuda semantics).
 *   Frames: device 8U with 1 to 256 interleaved channels (another depth: B2F_UNSUPPORTED_TYPE), pitched or an ROI.
 *   Pyramids (b2f_lkpyr_pyramid): device levels with a (win_w, win_h) border, BORDER_REFLECT_101 for the uint8 levels
 *      and BORDER_CONSTANT for the int16 Scharr derivatives (CV_16SC(2 cn), Ix and Iy per channel); other border modes
 *      are refused with B2F_UNSUPPORTED_TYPE (BORDER_ISOLATED is accepted and implied).  A pyramid grows on demand; a
 *      build that needs more memory first waits for its stream.  b2f_lkpyr_pyramid_level views a level, border
 *      included: rows + 2 win_h by cols + 2 win_w.
 *   b2f_lkpyr_calc: prev and next are each an image or a pyramid (exactly one of the two pointers).  A pyramid caps
 *      max_level at its own level count and must have a border of at least the window (else B2F_BAD_ARG); an image is
 *      built up to what is left.  prev_pts / next_pts: n_points interleaved (x, y) float32 on the device; status: n
 *      bytes; err: n float32 or NULL.  next_pts is read first only with B2F_LKPYR_USE_INITIAL_FLOW.  err is written where
 *      cv2 writes it (tracked points, points outside the image on level 0 (0), and every point that reached the
 *      covariance under B2F_LKPYR_GET_MIN_EIGENVALS); elsewhere the caller's values stay.  Everything runs on
 *      `cuda_stream` without host synchronisation (a NULL stream ends with a device synchronise); the first call at a
 *      new size waits for the stream while it lays out the handle's workspace.  A handle may be called on several
 *      streams: a call on another stream than the previous call first waits (on the device) for that call's work,
 *      since both share the handle's workspace.  A pyramid is the caller's memory: rebuilding it while a calc on
 *      another stream still reads it is the caller's race, and a rebuild at another size, channel count, window,
 *      level count or derivative choice moves its levels, so views taken before it are stale. ---- */
enum { B2F_LKPYR_USE_INITIAL_FLOW = 4, B2F_LKPYR_GET_MIN_EIGENVALS = 8 }; /* cv::OPTFLOW_USE_INITIAL_FLOW, OPTFLOW_LK_GET_MIN_EIGENVALS */
typedef struct b2f_lkpyr_params {
    int win_width;            /* 21 */
    int win_height;           /* 21 */
    int max_level;            /* 3  */
    int criteria_type;        /* 3: TermCriteria::COUNT (1) | TermCriteria::EPS (2) */
    int max_count;            /* 30 */
    double epsilon;           /* 0.01 */
    int flags;                /* 0  */
    double min_eig_threshold; /* 1e-4 */
} b2f_lkpyr_params;
typedef struct b2f_lkpyr b2f_lkpyr;
typedef struct b2f_lkpyr_pyramid b2f_lkpyr_pyramid;
B2F_API void b2f_lkpyr_default_params(b2f_lkpyr_params *p);
B2F_API int b2f_lkpyr_create(const b2f_lkpyr_params *p, b2f_lkpyr **out); /* NULL: the defaults */
B2F_API int b2f_lkpyr_set_params(b2f_lkpyr *h, const b2f_lkpyr_params *p);
B2F_API int b2f_lkpyr_get_params(const b2f_lkpyr *h, b2f_lkpyr_params *p);
/* borrowed base handle, for b2f_get_param(B2F_ENGINE_ACTIVE_PATH) and b2f_get_stats */
B2F_API b2f_handle *b2f_lkpyr_engine(b2f_lkpyr *h);
B2F_API int b2f_lkpyr_pyramid_create(b2f_lkpyr_pyramid **out);
B2F_API void b2f_lkpyr_pyramid_destroy(b2f_lkpyr_pyramid *p);
/* buildOpticalFlowPyramid: *max_level_out receives its return value (the last level built) */
B2F_API int b2f_lkpyr_build_pyramid(const b2f_image *img, int win_w, int win_h, int max_level, int with_derivatives,
                                    int pyr_border, int deriv_border, b2f_lkpyr_pyramid *pyr, int *max_level_out,
                                    void *cuda_stream);
B2F_API int b2f_lkpyr_pyramid_info(const b2f_lkpyr_pyramid *p, int *levels, int *win_w, int *win_h,
                                   int *with_derivatives);
B2F_API int b2f_lkpyr_pyramid_level(const b2f_lkpyr_pyramid *p, int level, int deriv, b2f_image *view);
B2F_API int b2f_lkpyr_calc(b2f_lkpyr *h, const b2f_image *prev_img, const b2f_lkpyr_pyramid *prev_pyr,
                           const b2f_image *next_img, const b2f_lkpyr_pyramid *next_pyr, const float *prev_pts,
                           float *next_pts, unsigned char *status, float *err, int n_points, void *cuda_stream);
B2F_API int b2f_lkpyr_last_cuda_error(const b2f_lkpyr *h);
B2F_API void b2f_lkpyr_destroy(b2f_lkpyr *h);

#ifdef __cplusplus
}
#endif
#endif /* B200FLOW_H_ */
