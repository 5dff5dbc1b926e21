"""BTV-L1 super-resolution model: ctypes driver of oracle/superres_model.c and the reference's pull schedule.
TEST INFRASTRUCTURE (see oracle/__init__.py).

``BTVL1`` transcribes BTVL1_CUDA's initImpl / processImpl / readNextFrame / processFrame (modules/superres/src/
btv_l1_cuda.cpp:483-582) and the ring buffer's ``at`` (src/ring_buffer.hpp:54-74) line for line; ``process`` calls the C
model.  One departure, as the engine makes it: with fewer than R + 1 frames the reference calls process with baseIdx -1
(out of bounds); here processFrame(idx) is skipped for idx > storePos.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_DIR, "superres_model.c")
_PATH = os.path.join(_DIR, "_build", "libsuperres_model.so")
_lib = None


def build(path: str = _PATH) -> str:
    """Compile the model to ``path`` with oracle/Makefile's flags (-ffp-contract=off: float only, no FMA contraction);
    ``__graft_entry__.build()`` calls this."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    subprocess.run(["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-fPIC", "-shared", "-o", path, _SRC, "-lm"],
                   check=True)
    return path


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} not built: run __graft_entry__.build()")
        l = C.CDLL(_PATH)
        vp, fp = C.c_void_p, C.POINTER(C.c_float)
        l.sr_model_gray.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        l.sr_model_gray.restype = None
        l.sr_model_gaussian_kernel.argtypes = [C.c_int, C.c_double, fp]
        l.sr_model_gaussian_kernel.restype = None
        l.sr_model_sep_filter.argtypes = [fp, C.c_int, C.c_int, C.c_int, fp, C.c_int, fp]
        l.sr_model_sep_filter.restype = None
        l.sr_model_process.argtypes = [fp, fp, fp] + [C.c_int] * 7 + [C.c_double] * 3 + [C.c_int, C.c_int, C.c_double, fp]
        l.sr_model_process.restype = C.c_int
        _lib = l
    return _lib


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


@dataclass
class Params:
    """BTVL1_CUDA's defaults (btv_l1_cuda.cpp:280-304, 459-462)."""
    scale: int = 4
    iterations: int = 180
    tau: float = 1.3
    lambda_: float = 0.03
    alpha: float = 0.7
    btv_kernel_size: int = 7
    blur_kernel_size: int = 5
    blur_sigma: float = 0.0
    temporal_area_radius: int = 4


def gray(frame: np.ndarray, to_f32: bool) -> np.ndarray:
    """The flow wrappers' conversion: BGR(A) -> gray by cudev's 15-bit rule, then x float(1/255) for a 32F work type."""
    a = np.ascontiguousarray(frame, np.uint8)
    cn = 1 if a.ndim == 2 else a.shape[2]
    out = np.empty(a.shape[:2], np.float32 if to_f32 else np.uint8)
    lib().sr_model_gray(a.ctypes.data, a.shape[0], a.shape[1], cn, int(to_f32), out.ctypes.data)
    return out


def gaussian_kernel(n: int, sigma: float) -> np.ndarray:
    out = np.empty(n, np.float32)
    lib().sr_model_gaussian_kernel(n, sigma, _fp(out))
    return out


def sep_filter(src: np.ndarray, n: int, sigma: float) -> np.ndarray:
    """cuda::createGaussianFilter(type, -1, (n, n), sigma)->apply on an H x W[ x C] float image."""
    a = np.ascontiguousarray(src, np.float32)
    cn = 1 if a.ndim == 2 else a.shape[2]
    k = gaussian_kernel(n, sigma)
    out = np.empty_like(a)
    lib().sr_model_sep_filter(_fp(a), a.shape[0], a.shape[1], cn, _fp(k), n, _fp(out))
    return out


def process(src, fwd, bwd, base: int, P: Params) -> np.ndarray:
    """BTVL1_CUDA_Base::process before the crop: src K frames H x W[ x C] float32, fwd[k] (u, v) flow k -> k + 1 (None for
    the last), bwd[k] flow k -> k - 1 (None for the first).  Returns the (H s) x (W s) x C estimate."""
    K = len(src)
    h, w = src[0].shape[:2]
    cn = 1 if src[0].ndim == 2 else src[0].shape[2]
    S = np.ascontiguousarray(np.stack([np.asarray(f, np.float32).reshape(h, w, cn) for f in src]))
    z = np.zeros((2, h, w), np.float32)
    F = np.ascontiguousarray(np.stack([z if f is None else np.stack([f[0], f[1]]).astype(np.float32) for f in fwd]))
    B = np.ascontiguousarray(np.stack([z if f is None else np.stack([f[0], f[1]]).astype(np.float32) for f in bwd]))
    hr = np.empty((h * P.scale, w * P.scale, cn), np.float32)
    rc = lib().sr_model_process(_fp(S), _fp(F), _fp(B), K, base, h, w, cn, P.scale, P.iterations, P.tau, P.lambda_,
                                P.alpha, P.btv_kernel_size, P.blur_kernel_size, P.blur_sigma, _fp(hr))
    if rc != 0:
        raise MemoryError("sr_model_process")
    return hr


def to_u8(a: np.ndarray) -> np.ndarray:
    """GpuMat::convertTo(CV_8U) of float: round half to even, saturate (NaN -> 0)."""
    return np.clip(np.nan_to_num(np.rint(a), nan=0.0), 0, 255).astype(np.uint8)


def at(index: int, items: list):
    """ring_buffer.hpp:54-74"""
    n = len(items)
    if index < 0:
        num = index - n + 1
        index -= (-((-num) // n) if num < 0 else num // n) * n  # C++ division truncates toward zero
    if index >= n:
        index %= n
    return index


class BTVL1:
    """BTVL1_CUDA's schedule over a frame source (``next_frame()`` returns an H x W[ x C] uint8 array or None) and a flow
    function ``flow(frame0, frame1) -> (u, v)`` on the raw frames.  ``next_frame()`` returns the cropped float output (the
    reference's nextFrame is ``to_u8`` of it) or None; ``log`` records (idx, startIdx, endIdx, baseIdx) per process."""

    def __init__(self, source, flow, P: Params | None = None):
        self.src, self.flow, self.P = source, flow, P or Params()
        self.first = True
        self.log = []

    def _init(self):
        R = self.P.temporal_area_radius
        cache = 2 * R + 1
        self.frames = [None] * cache
        self.fwd = [None] * cache
        self.bwd = [None] * cache
        self.outputs = [None] * cache
        self.store_pos = -1
        for _ in range(-R, R + 1):
            self._read()
        for i in range(R + 1):
            if i <= self.store_pos:  # departure: the reference processes idx > storePos with baseIdx -1
                self._process_frame(i)
        self.proc_pos = R
        self.out_pos = -1

    def next_frame(self):
        if self.first:
            self._init()
            self.first = False
        if self.out_pos >= self.store_pos:
            return None
        self._read()
        if self.proc_pos < self.store_pos:
            self.proc_pos += 1
            self._process_frame(self.proc_pos)
        self.out_pos += 1
        return self.outputs[at(self.out_pos, self.outputs)]

    def _read(self):
        cur = self.src.next_frame()
        if cur is None:
            return
        self.store_pos += 1
        self.frames[at(self.store_pos, self.frames)] = np.asarray(cur).astype(np.float32)
        if self.store_pos > 0:
            self.fwd[at(self.store_pos - 1, self.fwd)] = self.flow(self.prev, cur)
            self.bwd[at(self.store_pos, self.bwd)] = self.flow(cur, self.prev)
        self.prev = np.array(cur, copy=True)

    def _process_frame(self, idx):
        R = self.P.temporal_area_radius
        start = max(idx - R, 0)
        end = min(start + 2 * R, self.store_pos)
        src, fwd, bwd, base = [], [], [], -1
        for k, i in enumerate(range(start, end + 1)):
            if i == idx:
                base = k
            src.append(self.frames[at(i, self.frames)])
            fwd.append(self.fwd[at(i, self.fwd)] if i < end else None)
            bwd.append(self.bwd[at(i, self.bwd)] if i > start else None)
        self.log.append((idx, start, end, base))
        hr = process(src, fwd, bwd, base, self.P)
        b = self.P.btv_kernel_size
        out = hr[b:hr.shape[0] - b, b:hr.shape[1] - b]
        self.outputs[at(idx, self.outputs)] = out if out.shape[2] > 1 else out[..., 0]


class ListSource:
    def __init__(self, frames):
        self.frames, self.i = list(frames), 0

    def next_frame(self):
        if self.i >= len(self.frames):
            return None
        self.i += 1
        return self.frames[self.i - 1]


def run(frames, flow, P: Params | None = None):
    """Every output of a stream: a list of cropped float images."""
    m = BTVL1(ListSource(frames), flow, P)
    outs = []
    while True:
        o = m.next_frame()
        if o is None:
            return outs, m.log
        outs.append(np.array(o, copy=True))
