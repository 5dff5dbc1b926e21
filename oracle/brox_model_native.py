"""ctypes loader for oracle/brox_model.c, the C/OpenMP restatement of oracle/brox_model.py.
TEST INFRASTRUCTURE (see oracle/__init__.py).  Float only: it is bit-identical to the numpy model and, with
rsqrt="exact", to the engine with aux_path 1."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .brox_model import COUNTER_NAMES, RSQRT_MODES, BroxParams
from .tvl1_cpu_native import usable_cpus

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libbrox_model.so")
_lib = None


def available() -> bool:
    return os.path.exists(_PATH)


def lib():
    global _lib
    if _lib is None:
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        l = C.CDLL(_PATH)
        l.brox_model_set_threads.restype = C.c_int
        l.brox_model_set_threads.argtypes = [C.c_int]
        l.brox_model_set_threads(usable_cpus())
        l.brox_model_n_counters.restype = C.c_int
        assert l.brox_model_n_counters() == len(COUNTER_NAMES)
        fp = C.POINTER(C.c_float)
        l.brox_model_rsqrt_batch.restype = None
        l.brox_model_rsqrt_batch.argtypes = [fp, C.c_long, fp]
        l.brox_model_calc.restype = C.c_int
        l.brox_model_calc.argtypes = [fp, fp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                      C.c_int, C.c_int, fp, C.POINTER(C.c_longlong)]
        _lib = l
    return _lib


def rsqrt_rn(x: np.ndarray) -> np.ndarray:
    """The model's correctly rounded 1/sqrt (brox_model_rsqrt_rn) over an array of positive finite floats."""
    a = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(a)
    fp = C.POINTER(C.c_float)
    lib().brox_model_rsqrt_batch(a.ctypes.data_as(fp), a.size, out.ctypes.data_as(fp))
    return out


def calc(I0: np.ndarray, I1: np.ndarray, P: BroxParams | None = None, rsqrt="exact", counters=None) -> np.ndarray:
    """Same contract as oracle.brox_model.calc, counters included."""
    P = P or BroxParams()
    assert I0.dtype == np.float32 and I1.dtype == np.float32 and I0.shape == I1.shape
    a, b = np.ascontiguousarray(I0), np.ascontiguousarray(I1)
    h, w = a.shape
    flow = np.empty((h, w, 2), np.float32)
    cnt = (C.c_longlong * len(COUNTER_NAMES))()
    fp = C.POINTER(C.c_float)
    rc = lib().brox_model_calc(a.ctypes.data_as(fp), b.ctypes.data_as(fp), h, w, float(np.float32(P.alpha)),
                               float(np.float32(P.gamma)), float(np.float32(P.scale_factor)), int(P.inner_iterations),
                               int(P.outer_iterations), int(P.solver_iterations), RSQRT_MODES.index(rsqrt),
                               flow.ctypes.data_as(fp), cnt)
    if rc != 0:
        raise (MemoryError if rc == -1 else ValueError)(f"brox_model_calc returned {rc}")
    if counters is not None:
        counters.update(zip(COUNTER_NAMES, (int(c) for c in cnt)))
    return flow
