"""ctypes loader for oracle/tvl1_gpu_model.c, the C/OpenMP restatement of oracle/tvl1_gpu_model.py.
TEST INFRASTRUCTURE (see oracle/__init__.py).  Three builds of one source: precision "f32" is the reference's CUDA
semantics in float (bit-identical to the numpy model), "f64" the same algorithm in double, the yardstick for float
rounding, and "eng" the engine's own roundings, which the engine must equal bit for bit.  "eng" emulates
rcp.approx.ftz / sqrt.approx.ftz from tables of their device values: set_mufu_tables() before calc()."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .tvl1_cpu_native import usable_cpus

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATHS = {"f32": os.path.join(_HERE, "_build", "libtvl1_gpu_model_f32.so"),
          "f64": os.path.join(_HERE, "_build", "libtvl1_gpu_model_f64.so"),
          "eng": os.path.join(_HERE, "_build", "libtvl1_gpu_model_eng.so")}
_DTYPES = {"f32": np.float32, "f64": np.float64, "eng": np.float32}
RCP_ENTRIES, SQRT_ENTRIES = 1 << 23, 1 << 24  # mantissas of [1, 2); mantissa x exponent parity of [1, 4)
_libs: dict = {}


class _Params(C.Structure):
    _fields_ = [("tau", C.c_double), ("lambda_", C.c_double), ("theta", C.c_double), ("nscales", C.c_int),
                ("warps", C.c_int), ("epsilon", C.c_double), ("iterations", C.c_int), ("scaleStep", C.c_double),
                ("gamma", C.c_double), ("useInitialFlow", C.c_int), ("medianFiltering", C.c_int),
                ("medianPeriod", C.c_int)]


class _Trace(C.Structure):
    _fields_ = [("iters", C.POINTER(C.c_int)), ("iters_cap", C.c_int), ("n_iters", C.c_int),
                ("ratios", C.POINTER(C.c_double)), ("ratios_cap", C.c_int), ("n_ratios", C.c_int)]


def available(precision: str = "f32") -> bool:
    return os.path.exists(_PATHS[precision])


def lib(precision: str = "f32"):
    l = _libs.get(precision)
    if l is None:
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        l = C.CDLL(_PATHS[precision])
        l.tvl1_model_set_threads.restype = C.c_int
        l.tvl1_model_set_threads.argtypes = [C.c_int]
        l.tvl1_model_set_threads(usable_cpus())
        l.tvl1_model_real_bytes.restype = C.c_int
        assert l.tvl1_model_real_bytes() == np.dtype(_DTYPES[precision]).itemsize
        fp = C.POINTER(C.c_float)
        l.tvl1_model_calc.restype = C.c_int
        l.tvl1_model_calc.argtypes = [C.POINTER(_Params), fp, fp, C.c_int, C.c_int, C.c_int, fp, C.c_void_p,
                                      C.POINTER(_Trace)]
        l.tvl1_model_sum.restype = C.c_double
        l.tvl1_model_sum.argtypes = [C.c_void_p, C.c_long]
        l.tvl1_model_engine_rounding.restype = C.c_int
        assert l.tvl1_model_engine_rounding() == (precision == "eng")
        if precision == "eng":
            l.tvl1_model_set_mufu_tables.restype = C.c_int
            l.tvl1_model_set_mufu_tables.argtypes = [C.c_void_p, C.c_void_p]
            l.tvl1_model_mufu_apply.restype = C.c_int
            l.tvl1_model_mufu_apply.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_long]
        _libs[precision] = l
    return l


def set_threads(n: int, precision: str = "f32") -> int:
    return int(lib(precision).tvl1_model_set_threads(int(n)))


def set_mufu_tables(rcp: np.ndarray, sqrt: np.ndarray) -> None:
    """The "eng" build's rcp.approx table (2^23 float32: the values at the floats 0x3f800000 + m) and sqrt.approx table
    (2^24 float32: the values at 0x3f800000 + i, i = (exponent parity << 23) | m, i.e. all of [1, 4))."""
    rcp = np.ascontiguousarray(rcp, np.float32)
    sqrt = np.ascontiguousarray(sqrt, np.float32)
    assert rcp.shape == (RCP_ENTRIES,) and sqrt.shape == (SQRT_ENTRIES,)
    if lib("eng").tvl1_model_set_mufu_tables(rcp.ctypes.data, sqrt.ctypes.data) != 0:
        raise MemoryError("tvl1_model_set_mufu_tables")


def mufu_apply(op: int, x: np.ndarray) -> np.ndarray:
    """The "eng" build's emulation of rcp.approx.ftz (op 0) / sqrt.approx.ftz (op 1), element-wise on float32."""
    a = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(a)
    if lib("eng").tvl1_model_mufu_apply(int(op), a.ctypes.data, out.ctypes.data, a.size) != 0:
        raise RuntimeError("MUFU tables not set: call set_mufu_tables() first")
    return out


def error_sum(err: np.ndarray, precision: str = "f32") -> float:
    """The model's sum of an error image (numpy's pairwise order, in double)."""
    a = np.ascontiguousarray(err, _DTYPES[precision])
    return float(lib(precision).tvl1_model_sum(a.ctypes.data, a.size))


def calc(I0: np.ndarray, I1: np.ndarray, P=None, init_flow=None, trace=None, ratios=None,
         precision: str = "f32", median=(1, 0)) -> np.ndarray:
    """Same contract as oracle.tvl1_gpu_model.calc (P: its TVL1Params).  Returns (H, W, 2) flow in float32 ("f32",
    "eng") or float64 ("f64").  trace: list, receives one list of per-warp inner-iteration counts per solved level
    (coarsest first).  ratios: list, receives every sampled error sum over its level's scaledEpsilon, in order.
    median: (kernel size 1 / 3 / 5, period) -- the engine's MEDIAN_FILTERING / MEDIAN_PERIOD knobs."""
    from .tvl1_gpu_model import TVL1Params
    P = P or TVL1Params()
    assert I0.dtype in (np.uint8, np.float32) and I0.shape == I1.shape and I0.dtype == I1.dtype
    h, w = I0.shape
    a = np.ascontiguousarray(I0, np.float32)
    b = np.ascontiguousarray(I1, np.float32)
    init = None
    if P.useInitialFlow:
        init = np.ascontiguousarray(init_flow, np.float32)
        assert init.shape == (h, w, 2)
    flow = np.empty((h, w, 2), _DTYPES[precision])
    p = _Params(P.tau, P.lambda_, P.theta, P.nscales, P.warps, P.epsilon, P.iterations, P.scaleStep, P.gamma,
                int(P.useInitialFlow), int(median[0]), int(median[1]))
    cap_i = max(1, P.nscales * P.warps)
    iters = (C.c_int * cap_i)()
    cap_r = max(1, P.nscales * P.warps * (P.iterations // 2 + 1))
    rbuf = (C.c_double * cap_r)()
    tr = _Trace(iters, cap_i, 0, rbuf, cap_r, 0)
    fp = lambda x: None if x is None else x.ctypes.data_as(C.POINTER(C.c_float))
    rc = lib(precision).tvl1_model_calc(C.byref(p), fp(a), fp(b), h, w, int(I0.dtype == np.uint8), fp(init),
                                        flow.ctypes.data, C.byref(tr))
    if rc != 0:
        if rc == -3:
            raise RuntimeError("MUFU tables not set: call set_mufu_tables() first")
        raise (MemoryError if rc == -1 else ValueError)(f"tvl1_model_calc returned {rc}")
    if trace is not None:
        counts = list(iters[:tr.n_iters])
        trace.extend(counts[i:i + P.warps] for i in range(0, len(counts), max(1, P.warps)))
    if ratios is not None:
        ratios.extend(rbuf[:tr.n_ratios])
    return flow
