"""ctypes loader for libb200flow.so (the C ABI in include/b200flow.h).

The library is built in-tree by ``__graft_entry__.build()`` (or ``make -C
opencv_contrib_b200/csrc``).  There is no CPU fallback: if the shared object is
missing or a CUDA call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200flow.so")

B2F_OK = 0
B2F_8UC1, B2F_32FC1, B2F_32FC2 = 0, 5, 13
B2F_MAX_KERNEL_CLASSES = 16

STATUS_NAMES = {0: "B2F_OK", 1: "B2F_BAD_ARG", 2: "B2F_UNSUPPORTED_TYPE", 3: "B2F_SIZE_MISMATCH",
                4: "B2F_CUDA_ERROR", 5: "B2F_NO_DEVICE", 6: "B2F_OUT_OF_MEMORY"}


class b2f_image(C.Structure):
    _fields_ = [("data", C.c_void_p), ("step", C.c_size_t), ("rows", C.c_int), ("cols", C.c_int),
                ("type", C.c_int)]


class b2f_tvl1_params(C.Structure):
    _fields_ = [("tau", C.c_double), ("lambda_", C.c_double), ("theta", C.c_double),
                ("nscales", C.c_int), ("warps", C.c_int), ("epsilon", C.c_double),
                ("iterations", C.c_int), ("scale_step", C.c_double), ("gamma", C.c_double),
                ("use_initial_flow", C.c_int)]


class b2f_farneback_params(C.Structure):
    _fields_ = [("num_levels", C.c_int), ("pyr_scale", C.c_double), ("fast_pyramids", C.c_int),
                ("win_size", C.c_int), ("num_iters", C.c_int), ("poly_n", C.c_int),
                ("poly_sigma", C.c_double), ("flags", C.c_int)]


class b2f_brox_params(C.Structure):
    _fields_ = [("alpha", C.c_double), ("gamma", C.c_double), ("scale_factor", C.c_double),
                ("inner_iterations", C.c_int), ("outer_iterations", C.c_int),
                ("solver_iterations", C.c_int)]


class b2f_denselk_params(C.Structure):
    _fields_ = [("win_width", C.c_int), ("win_height", C.c_int), ("max_level", C.c_int),
                ("iters", C.c_int), ("use_initial_flow", C.c_int)]


class b2f_deepflow_params(C.Structure):
    _fields_ = [("sigma", C.c_double), ("min_size", C.c_int), ("downscale_factor", C.c_double),
                ("fixed_point_iterations", C.c_int), ("sor_iterations", C.c_int), ("alpha", C.c_double),
                ("delta", C.c_double), ("gamma", C.c_double), ("omega", C.c_double), ("max_layers", C.c_int)]


class b2f_dis_params(C.Structure):
    _fields_ = [("finest_scale", C.c_int), ("coarsest_scale", C.c_int), ("patch_size", C.c_int),
                ("patch_stride", C.c_int), ("grad_descent_iterations", C.c_int),
                ("variational_refinement_iterations", C.c_int), ("alpha", C.c_double), ("delta", C.c_double),
                ("gamma", C.c_double), ("epsilon", C.c_double), ("use_mean_normalization", C.c_int),
                ("use_spatial_propagation", C.c_int), ("use_initial_flow", C.c_int)]


class b2f_fastbm_params(C.Structure):
    _fields_ = [("search_window", C.c_int), ("block_window", C.c_int)]


class b2f_varref_params(C.Structure):
    _fields_ = [("fixed_point_iterations", C.c_int), ("sor_iterations", C.c_int), ("omega", C.c_double),
                ("alpha", C.c_double), ("delta", C.c_double), ("gamma", C.c_double), ("epsilon", C.c_double)]


class b2f_sparselk_params(C.Structure):
    _fields_ = [("win_width", C.c_int), ("win_height", C.c_int), ("max_level", C.c_int), ("iters", C.c_int),
                ("use_initial_flow", C.c_int)]


class b2f_superres_params(C.Structure):
    _fields_ = [("scale", C.c_int), ("iterations", C.c_int), ("tau", C.c_double), ("lambda_", C.c_double),
                ("alpha", C.c_double), ("btv_kernel_size", C.c_int), ("blur_kernel_size", C.c_int),
                ("blur_sigma", C.c_double), ("temporal_area_radius", C.c_int)]


class b2f_gftt_params(C.Structure):
    _fields_ = [("max_corners", C.c_int), ("quality_level", C.c_double), ("min_distance", C.c_double),
                ("block_size", C.c_int), ("use_harris", C.c_int), ("harris_k", C.c_double)]


class b2f_gftt_info(C.Structure):
    _fields_ = [("candidates", C.c_int), ("kept", C.c_int), ("capped", C.c_int), ("rounds", C.c_int)]


class b2f_lkpyr_params(C.Structure):
    _fields_ = [("win_width", C.c_int), ("win_height", C.c_int), ("max_level", C.c_int), ("criteria_type", C.c_int),
                ("max_count", C.c_int), ("epsilon", C.c_double), ("flags", C.c_int), ("min_eig_threshold", C.c_double)]


class b2f_stats(C.Structure):
    _fields_ = [("calls", C.c_uint64), ("launches", C.c_uint64),
                ("class_launches", C.c_uint64 * B2F_MAX_KERNEL_CLASSES),
                ("class_ms", C.c_double * B2F_MAX_KERNEL_CLASSES),
                ("class_bytes", C.c_double * B2F_MAX_KERNEL_CLASSES),
                ("levels", C.c_int), ("iterations_run", C.c_int)]


class b2f_error_stats(C.Structure):
    _fields_ = [("mean", C.c_double), ("stddev", C.c_double), ("r", C.c_double * 5), ("a", C.c_double * 3),
                ("max", C.c_double), ("count", C.c_int64)]


# every symbol include/b200flow.h declares: (name, restype, argtypes)
_H = C.c_void_p
_IMG = C.POINTER(b2f_image)
_F = C.POINTER(C.c_float)
SYMBOLS = [
    ("b2f_tvl1_default_params", None, [C.POINTER(b2f_tvl1_params)]),
    ("b2f_farneback_default_params", None, [C.POINTER(b2f_farneback_params)]),
    ("b2f_brox_default_params", None, [C.POINTER(b2f_brox_params)]),
    ("b2f_denselk_default_params", None, [C.POINTER(b2f_denselk_params)]),
    ("b2f_deepflow_default_params", None, [C.POINTER(b2f_deepflow_params)]),
    ("b2f_dis_default_params", None, [C.POINTER(b2f_dis_params), C.c_int]),
    ("b2f_tvl1_create", C.c_int, [C.POINTER(b2f_tvl1_params), C.POINTER(_H)]),
    ("b2f_median_blur_32f", C.c_int, [C.POINTER(b2f_image), C.POINTER(b2f_image), C.c_int, C.c_void_p]),
    ("b2f_approx_probe", C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("b2f_farneback_create", C.c_int, [C.POINTER(b2f_farneback_params), C.POINTER(_H)]),
    ("b2f_brox_create", C.c_int, [C.POINTER(b2f_brox_params), C.POINTER(_H)]),
    ("b2f_denselk_create", C.c_int, [C.POINTER(b2f_denselk_params), C.POINTER(_H)]),
    ("b2f_deepflow_create", C.c_int, [C.POINTER(b2f_deepflow_params), C.POINTER(_H)]),
    ("b2f_dis_create", C.c_int, [C.POINTER(b2f_dis_params), C.POINTER(_H)]),
    ("b2f_fastbm_default_params", None, [C.POINTER(b2f_fastbm_params)]),
    ("b2f_fastbm_create", C.c_int, [C.POINTER(b2f_fastbm_params), C.POINTER(_H)]),
    ("b2f_varref_default_params", None, [C.POINTER(b2f_varref_params)]),
    ("b2f_varref_create", C.c_int, [C.POINTER(b2f_varref_params), C.POINTER(_H)]),
    ("b2f_optflowgf_create", C.c_int, [C.POINTER(b2f_farneback_params), C.POINTER(_H)]),
    ("b2f_calc_optical_flow_bm_size", C.c_int, [C.c_int] * 8 + [C.POINTER(C.c_int)] * 3),
    ("b2f_calc_optical_flow_bm", C.c_int, [_IMG, _IMG] + [C.c_int] * 7 + [_IMG, _IMG, C.c_void_p]),
    ("b2f_destroy", None, [_H]),
    ("b2f_set_param", C.c_int, [_H, C.c_int, C.c_double]),
    ("b2f_get_param", C.c_int, [_H, C.c_int, C.POINTER(C.c_double)]),
    ("b2f_default_name", C.c_char_p, [_H]),
    ("b2f_calc", C.c_int, [_H, C.POINTER(b2f_image), C.POINTER(b2f_image), C.POINTER(b2f_image), C.c_void_p]),
    ("b2f_calc_host", C.c_int, [_H, C.POINTER(b2f_image), C.POINTER(b2f_image), C.POINTER(b2f_image), C.c_void_p]),
    ("b2f_workspace_bytes", C.c_size_t, [_H, C.c_int, C.c_int, C.c_int]),
    ("b2f_status_string", C.c_char_p, [C.c_int]),
    ("b2f_last_cuda_error", C.c_int, [_H]),
    ("b2f_version", C.c_char_p, []),
    ("b2f_get_stats", C.c_int, [_H, C.POINTER(b2f_stats)]),
    ("b2f_reset_stats", C.c_int, [_H]),
    ("b2f_kernel_class_name", C.c_char_p, [_H, C.c_int]),
    ("b2f_set_profiling", C.c_int, [_H, C.c_int]),
    # adjacent components (SURVEY 8f)
    ("b2f_calc_uv", C.c_int, [_H, _IMG, _IMG, _IMG, _IMG, C.c_void_p]),
    ("b2f_interpolate_frames", C.c_int, [_IMG, _IMG, _IMG, _IMG, _IMG, _IMG, C.c_float, _IMG, _IMG, C.c_int,
                                         C.c_void_p]),
    ("b2f_video_create", C.c_int, [_H, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_H)]),
    ("b2f_video_push", C.c_int, [_H, C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)]),
    ("b2f_video_fetch", C.c_int, [_H, C.c_int64, C.c_void_p, C.c_size_t]),
    ("b2f_video_fetch_view", C.c_int, [_H, C.c_int64, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_size_t)]),
    ("b2f_video_destroy", None, [_H]),
    ("b2f_sparselk_default_params", None, [C.POINTER(b2f_sparselk_params)]),
    ("b2f_sparselk_create", C.c_int, [C.POINTER(b2f_sparselk_params), C.POINTER(_H)]),
    ("b2f_sparselk_set_params", C.c_int, [_H, C.POINTER(b2f_sparselk_params)]),
    ("b2f_sparselk_get_params", C.c_int, [_H, C.POINTER(b2f_sparselk_params)]),
    ("b2f_sparselk_calc", C.c_int, [_H, _IMG, _IMG, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_void_p]),
    ("b2f_sparselk_destroy", None, [_H]),
    ("b2f_batch_create", C.c_int, [C.c_int, C.c_void_p, C.c_int, C.POINTER(_H)]),
    ("b2f_batch_streams", C.c_int, [_H]),
    ("b2f_batch_engine", C.c_void_p, [_H, C.c_int]),
    ("b2f_batch_set_param", C.c_int, [_H, C.c_int, C.c_double]),
    ("b2f_batch_run_device", C.c_int, [_H, C.c_int, _IMG, _IMG, _IMG, C.c_void_p]),
    ("b2f_batch_run_host", C.c_int, [_H, C.c_int, _IMG, _IMG, _IMG]),
    ("b2f_batch_run_device_gather", C.c_int, [_H, C.c_int, _IMG, _IMG, _IMG, _H, C.c_int, _IMG, C.c_void_p]),
    ("b2f_comm_available", C.c_int, []),
    ("b2f_comm_unique_id", C.c_int, [C.c_void_p, C.c_size_t]),
    ("b2f_comm_create", C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(_H)]),
    ("b2f_comm_adopt", C.c_int, [C.c_void_p, C.POINTER(_H)]),
    ("b2f_comm_rank", C.c_int, [_H]),
    ("b2f_comm_nranks", C.c_int, [_H]),
    ("b2f_comm_last_nccl_error", C.c_int, [_H]),
    ("b2f_comm_destroy", None, [_H]),
    ("b2f_batch_launches", C.c_uint64, [_H]),
    ("b2f_batch_reset_stats", C.c_int, [_H]),
    ("b2f_batch_destroy", None, [_H]),
    ("b2f_superres_default_params", None, [C.POINTER(b2f_superres_params)]),
    ("b2f_superres_create", C.c_int, [C.POINTER(b2f_superres_params), _H, C.POINTER(_H)]),
    ("b2f_superres_set_flow", C.c_int, [_H, _H]),
    ("b2f_superres_set_param", C.c_int, [_H, C.c_int, C.c_double]),
    ("b2f_superres_get_param", C.c_int, [_H, C.c_int, C.POINTER(C.c_double)]),
    ("b2f_superres_wants_frame", C.c_int, [_H, C.POINTER(C.c_int)]),
    ("b2f_superres_push", C.c_int, [_H, _IMG, C.c_void_p]),
    ("b2f_superres_push_flows", C.c_int, [_H, _IMG, _IMG, _IMG, _IMG, _IMG, C.c_void_p]),
    ("b2f_superres_pop", C.c_int, [_H, _IMG, C.POINTER(C.c_int), C.c_void_p]),
    ("b2f_superres_output_size", C.c_int, [_H, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("b2f_superres_reset", C.c_int, [_H]),
    ("b2f_superres_collect_garbage", C.c_int, [_H]),
    ("b2f_superres_get_stats", C.c_int, [_H, C.POINTER(b2f_stats)]),
    ("b2f_superres_reset_stats", C.c_int, [_H]),
    ("b2f_superres_last_cuda_error", C.c_int, [_H]),
    ("b2f_superres_destroy", None, [_H]),
    ("b2f_calc_ext", C.c_int, [_H, _IMG, _IMG, _IMG, _IMG, C.c_void_p]),
    ("b2f_harris_create", C.c_int, [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.POINTER(_H)]),
    ("b2f_mineig_create", C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_H)]),
    ("b2f_corners_compute", C.c_int, [_H, _IMG, _IMG, C.c_void_p]),
    ("b2f_gftt_default_params", None, [C.POINTER(b2f_gftt_params)]),
    ("b2f_gftt_create", C.c_int, [C.c_int, C.POINTER(b2f_gftt_params), C.POINTER(_H)]),
    ("b2f_gftt_set_params", C.c_int, [_H, C.POINTER(b2f_gftt_params)]),
    ("b2f_gftt_get_params", C.c_int, [_H, C.POINTER(b2f_gftt_params)]),
    ("b2f_gftt_capacity", C.c_int, [_H, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    ("b2f_gftt_detect", C.c_int, [_H, _IMG, _IMG, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    ("b2f_gftt_last_info", C.c_int, [_H, C.POINTER(b2f_gftt_info), C.c_void_p]),
    ("b2f_corners_last_cuda_error", C.c_int, [_H]),
    ("b2f_corners_destroy", None, [_H]),
    ("b2f_lkpyr_default_params", None, [C.POINTER(b2f_lkpyr_params)]),
    ("b2f_lkpyr_create", C.c_int, [C.POINTER(b2f_lkpyr_params), C.POINTER(_H)]),
    ("b2f_lkpyr_set_params", C.c_int, [_H, C.POINTER(b2f_lkpyr_params)]),
    ("b2f_lkpyr_get_params", C.c_int, [_H, C.POINTER(b2f_lkpyr_params)]),
    ("b2f_lkpyr_engine", C.c_void_p, [_H]),
    ("b2f_lkpyr_pyramid_create", C.c_int, [C.POINTER(_H)]),
    ("b2f_lkpyr_pyramid_destroy", None, [_H]),
    ("b2f_lkpyr_build_pyramid", C.c_int, [_IMG, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _H,
                                          C.POINTER(C.c_int), C.c_void_p]),
    ("b2f_lkpyr_pyramid_info", C.c_int, [_H] + [C.POINTER(C.c_int)] * 4),
    ("b2f_lkpyr_pyramid_level", C.c_int, [_H, C.c_int, C.c_int, _IMG]),
    ("b2f_lkpyr_calc", C.c_int, [_H, _IMG, _H, _IMG, _H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                 C.c_void_p]),
    ("b2f_lkpyr_last_cuda_error", C.c_int, [_H]),
    ("b2f_lkpyr_destroy", None, [_H]),
    ("b2f_flo_read_size", C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("b2f_flo_read", C.c_int, [C.c_char_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int]),
    ("b2f_flo_write", C.c_int, [C.c_char_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int]),
    ("b2f_flow_error_map", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_size_t]),
    ("b2f_flow_error_stats", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int,
                                       C.POINTER(b2f_error_stats)]),
    ("b2f_flow_accuracy", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_double,
                                    C.POINTER(C.c_double)]),
]

# b2f_param_id values (include/b200flow.h)
PARAM = {
    "tvl1": dict(tau=100, lambda_=101, theta=102, nscales=103, warps=104, epsilon=105, iterations=106,
                 scale_step=107, gamma=108, use_initial_flow=109,
                 median_filtering=120, median_period=121, initial_flow_source=122),
    "farneback": dict(num_levels=200, pyr_scale=201, fast_pyramids=202, win_size=203, num_iters=204,
                      poly_n=205, poly_sigma=206, flags=207),
    "brox": dict(alpha=300, gamma=301, scale_factor=302, inner_iterations=303, outer_iterations=304,
                 solver_iterations=305),
    "denselk": dict(win_width=400, win_height=401, max_level=402, iters=403, use_initial_flow=404),
    "deepflow": dict(sigma=500, min_size=501, downscale_factor=502, fixed_point_iterations=503, sor_iterations=504,
                     alpha=505, delta=506, gamma=507, omega=508, max_layers=509),
    "dis": dict(finest_scale=600, coarsest_scale=601, patch_size=602, patch_stride=603, grad_descent_iterations=604,
                variational_refinement_iterations=605, alpha=606, delta=607, gamma=608, epsilon=609,
                use_mean_normalization=610, use_spatial_propagation=611, use_initial_flow=612),
    "fastbm": dict(search_window=700, block_window=701),
    "varref": dict(fixed_point_iterations=950, sor_iterations=951, omega=952, alpha=953, delta=954, gamma=955,
                   epsilon=956),
    "superres": dict(scale=800, iterations=801, tau=802, lambda_=803, alpha=804, btv_kernel_size=805,
                     blur_kernel_size=806, blur_sigma=807, temporal_area_radius=808),
    "engine": dict(fused_iters=900, use_graph=901, kernel_path=902, aux_path=903, active_path=1000),
}
# b2f_tvl1_path flags (include/b200flow.h)
TVL1_PATH = dict(iter_tma=1, iter_blocked=2, iter_unfused=4, warp_tiled=8, warp_untiled=16)
# b2f_farneback_path values (include/b200flow.h)
FARN_PATH = dict(tma=1, quad=2, quad_wide=3, quad_r80=4, quad_r64=5, quad_transposed=6, fast=7, generic=8)
# b2f_brox_path values (include/b200flow.h); B2F_ENGINE_ACTIVE_PATH carries one in bits 0-7, iterations per launch in 8-15
BROX_PATH = dict(reg=1, smem=2, half_sweep=3, coop=4)

_lib = None


class B2FError(RuntimeError):
    def __init__(self, status: int, cuda_error: int = 0):
        self.status = status
        self.cuda_error = cuda_error
        msg = STATUS_NAMES.get(status, str(status))
        if _lib is not None:
            msg = _lib.b2f_status_string(status).decode()
        if cuda_error:
            msg += f" (cudaError {cuda_error})"
        super().__init__(msg)


def lib() -> C.CDLL:
    """Load libb200flow.so and bind every declared symbol.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)")
    l = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(l, name)  # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    _lib = l
    return l
