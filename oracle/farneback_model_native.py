"""ctypes loader for oracle/farneback_model.c, the C/OpenMP restatement of oracle/farneback_gpu_model.calc.
TEST INFRASTRUCTURE (see oracle/__init__.py).

Builds (oracle/Makefile):
* "f32"  -- the numpy float model in C, bit for bit equal to farneback_gpu_model.calc(precision="f32");
* "eng"  -- the engine's roundings (FMA contraction as the SASS shows it, the running box sum of the K = 6 iteration
  kernels, pyr_tap5 pyramids, the fused resize, skipped zero-weight level-image taps, the floor clamp): the model the
  Farneback engine must equal bit for bit;
* "only_<SWITCH>" -- f32 with one of those departures switched on (SWITCHES), so each can be seen to matter.

The iteration order ("fast" for the K = 6 register-blocked and TMA kernels, "generic" for k_farn_iter) follows the
engine's dispatch: order_for(P, kernel_path).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import farneback_gpu_model as fm
from .tvl1_cpu_native import usable_cpus

F = np.float32
SWITCHES = ("FMA", "RUNNING_BOX", "PYR_TAP5", "FUSED_RESIZE", "SKIP_ZERO", "FLOOR_CLAMP")
ORDERS = {"fast": 0, "generic": 1}
_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build")
_libs = {}


def _path(build):
    return os.path.join(_DIR, f"libfarneback_model_{build}.so")


def available(build="eng") -> bool:
    return os.path.exists(_path(build))


def lib(build="eng"):
    if build not in _libs:
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        l = C.CDLL(_path(build))
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
        l.farneback_model_set_threads.restype = C.c_int
        l.farneback_model_set_threads.argtypes = [C.c_int]
        l.farneback_model_set_threads(usable_cpus())
        l.farneback_model_switches.restype = C.c_int
        l.farneback_model_calc.restype = C.c_int
        l.farneback_model_calc.argtypes = [fp, fp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, fp, fp, ip, fp, fp, fp, C.c_int, fp]
        l.farneback_model_level_image.restype = C.c_int
        l.farneback_model_level_image.argtypes = [fp, C.c_int, C.c_int, fp, C.c_int, C.c_int, C.c_int, fp]
        l.farneback_model_box.restype = None
        l.farneback_model_box.argtypes = [fp, C.c_int, C.c_int, C.c_int, C.c_int, fp]
        _libs[build] = l
    return _libs[build]


def set_threads(n: int, build="eng") -> int:
    return lib(build).farneback_model_set_threads(int(n))


def order_for(P: fm.FarnebackParams, kernel_path: int = 0) -> str:
    """The engine runs the register-blocked (and TMA) iteration kernels for winSize 13 unless kernel_path is 1."""
    return "fast" if P.winSize // 2 == 6 and kernel_path != 1 else "generic"


def _poly_tabs(P):
    """The polynomial-expansion constants of farneback_gpu_model.prepare_gaussian.  The engine inverts the same 6x6
    matrix through Cholesky instead of LU; the float tables come out identical (checked for polyN 5 and 7 across sigma)."""
    t = fm.prepare_gaussian(P.polyN, P.polySigma)
    out = np.zeros(28, F)
    for i in range(3):
        out[8 * i:8 * i + P.polyN + 1] = t[i]
    out[24:28] = t[3:7]
    return out


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def calc(I0: np.ndarray, I1: np.ndarray, P: fm.FarnebackParams | None = None, init_flow=None, build="eng",
         order="fast") -> np.ndarray:
    """Same contract as farneback_gpu_model.calc (precision "f32"), in the rounding of `build`; order: "fast" or
    "generic" (see order_for)."""
    P = P or fm.FarnebackParams()
    assert P.polyN in (5, 7) and I0.shape == I1.shape
    a = np.ascontiguousarray(I0, F)
    b = np.ascontiguousarray(I1, F)
    h, w = a.shape
    sizes = fm.level_sizes(h, w, P)
    img_taps, offs = [], [0]
    for k in range(len(sizes)):
        scale = 1.0
        for _ in range(k):
            scale *= P.pyrScale
        sigma = (1.0 / scale - 1) * 0.5
        smooth = max(fm.cv_round(sigma * 5) | 1, 3)
        img_taps.append(fm.gaussian_kernel_half(smooth, sigma))
        offs.append(offs[-1] + len(img_taps[-1]))
    img_taps = np.ascontiguousarray(np.concatenate(img_taps), F)
    offs = (C.c_int * len(offs))(*offs)
    win = fm.gaussian_kernel_half(P.winSize, float(F(P.winSize // 2 * F(0.3))))
    win = np.ascontiguousarray(win, F)
    pyr = None
    if P.fastPyramids and not (lib(build).farneback_model_switches() & 4):
        levels = []
        for f in (a, b):
            cur = f
            for _ in range(1, len(sizes)):
                cur = fm.pyr_down(cur)
                levels.append(cur.ravel())
        pyr = np.ascontiguousarray(np.concatenate(levels), F) if levels else np.zeros(1, F)
    init = None
    if P.flags & fm.OPTFLOW_USE_INITIAL_FLOW:
        init = np.ascontiguousarray(init_flow, F)
        assert init.shape == (h, w, 2)
    tabs = _poly_tabs(P)
    flow = np.empty((h, w, 2), F)
    rc = lib(build).farneback_model_calc(_fp(a), _fp(b), h, w, P.numLevels, P.pyrScale, int(bool(P.fastPyramids)),
                                         P.winSize, P.numIters, P.polyN, P.flags, _fp(tabs), _fp(img_taps), offs,
                                         _fp(win), None if pyr is None else _fp(pyr),
                                         None if init is None else _fp(init), ORDERS[order], _fp(flow))
    if rc != 0:
        raise (MemoryError if rc == -1 else ValueError)(f"farneback_model_calc returned {rc}")
    return flow


def level_image(src: np.ndarray, taps: np.ndarray, h: int, w: int, build="eng") -> np.ndarray:
    """The level image of one frame: REFLECT101 blur with the half kernel `taps`, then the bilinear resize to h x w."""
    s = np.ascontiguousarray(src, F)
    t = np.ascontiguousarray(taps, F)
    out = np.empty((h, w), F)
    rc = lib(build).farneback_model_level_image(_fp(s), s.shape[0], s.shape[1], _fp(t), len(t) - 1, h, w, _fp(out))
    if rc != 0:
        raise MemoryError("farneback_model_level_image")
    return out


def box(M: np.ndarray, win_size: int, order="fast", build="eng") -> np.ndarray:
    """The box window of the iteration kernels over the 5 planes of M (5, h, w), replicate border, scaled by 1/area."""
    m = np.ascontiguousarray(M, F)
    out = np.empty_like(m)
    lib(build).farneback_model_box(_fp(m), m.shape[1], m.shape[2], int(win_size), ORDERS[order], _fp(out))
    return out
