"""Python mirror of the reference's generated cudaoptflow bindings.

Reference interface (modules/cudaoptflow/include/opencv2/cudaoptflow.hpp, wrapped for Python by
``WRAP python`` in modules/cudaoptflow/CMakeLists.txt:9):

    alg = cv2.cuda.OpticalFlowDual_TVL1_create(tau, lambda_, theta, nscales, warps, epsilon,
                                               iterations, scaleStep, gamma, useInitialFlow)
    flow = alg.calc(I0, I1, flow[, stream])          # GpuMat in, GpuMat CV_32FC2 out
    alg.getTau() / alg.setTau(v) ...                 # cudaoptflow.hpp:311-373

Here a ``GpuMat`` is a CUDA ``torch.Tensor`` (H x W uint8/float32 for images, H x W x 2 float32
for flow; row pitch may exceed the width) and a ``Stream`` is a ``torch.cuda.Stream``.  torch is
plumbing only (device memory + streams); all compute happens in libb200flow.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import (B2F_8UC1, B2F_32FC1, B2F_32FC2, B2FError, b2f_image, b2f_stats, PARAM)

OPTFLOW_USE_INITIAL_FLOW = 4
OPTFLOW_FARNEBACK_GAUSSIAN = 256


def _torch():
    import torch
    return torch


def _image_from_tensor(t, flow: bool = False) -> b2f_image:
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("expected a CUDA torch.Tensor (the GpuMat stand-in)")
    if flow:
        if t.dim() != 3 or t.shape[2] != 2 or t.dtype != torch.float32:
            raise B2FError(2)
        if t.stride(2) != 1 or t.stride(1) != 2:
            raise ValueError("flow tensor must be interleaved (H, W, 2) with contiguous pixels")
        return b2f_image(t.data_ptr(), t.stride(0) * 4, t.shape[0], t.shape[1], B2F_32FC2)
    if t.dim() != 2:
        raise B2FError(2)  # reference: CV_Assert(channels == 1)
    if t.stride(1) != 1:
        raise ValueError("image rows must be contiguous")
    if t.dtype == torch.uint8:
        return b2f_image(t.data_ptr(), t.stride(0), t.shape[0], t.shape[1], B2F_8UC1)
    if t.dtype == torch.float32:
        return b2f_image(t.data_ptr(), t.stride(0) * 4, t.shape[0], t.shape[1], B2F_32FC1)
    raise B2FError(2)


def _image_from_numpy(a: np.ndarray, flow: bool = False) -> b2f_image:
    if flow:
        if a.ndim != 3 or a.shape[2] != 2 or a.dtype != np.float32 or a.strides[2] != 4 or a.strides[1] != 8:
            raise B2FError(2)
        return b2f_image(a.ctypes.data, a.strides[0], a.shape[0], a.shape[1], B2F_32FC2)
    if a.ndim != 2 or a.strides[1] != a.itemsize:
        raise B2FError(2)
    if a.dtype == np.uint8:
        return b2f_image(a.ctypes.data, a.strides[0], a.shape[0], a.shape[1], B2F_8UC1)
    if a.dtype == np.float32:
        return b2f_image(a.ctypes.data, a.strides[0], a.shape[0], a.shape[1], B2F_32FC1)
    raise B2FError(2)


class DenseOpticalFlow:
    """cv::cuda::DenseOpticalFlow (cudaoptflow.hpp:70-81)."""

    _family = ""

    def _needs_initial_flow(self) -> bool:
        """True when calc() reads the caller's flow first (useInitialFlow / OPTFLOW_USE_INITIAL_FLOW)."""
        return False

    def __init__(self, handle):
        self._h = handle
        self._lib = _lib.lib()

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b2f_destroy(h)

    # -- cv::Algorithm
    def getDefaultName(self) -> str:
        return self._lib.b2f_default_name(self._h).decode()

    # -- the hot call
    def calc(self, I0, I1, flow=None, stream=None):
        """calc(I0, I1, flow[, stream]) -> flow  (cudaoptflow.hpp:80).  Asynchronous on ``stream``."""
        torch = _torch()
        if flow is None:
            if self._needs_initial_flow():  # the reference asserts a valid flow of matching size (tvl1flow.cpp:190)
                raise B2FError(1)
            flow = torch.empty((I0.shape[0], I0.shape[1], 2), dtype=torch.float32, device=I0.device)
        i0, i1, fl = _image_from_tensor(I0), _image_from_tensor(I1), _image_from_tensor(flow, True)
        if stream is None:
            stream = torch.cuda.current_stream(I0.device)
        sptr = stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)
        st = self._lib.b2f_calc(self._h, C.byref(i0), C.byref(i1), C.byref(fl), C.c_void_p(sptr))
        if st != 0:
            raise B2FError(st, self._lib.b2f_last_cuda_error(self._h))
        return flow

    def calcUV(self, I0, I1, u=None, v=None, stream=None):
        """Planar variant: calc + cuda::split in one call (b2f_calc_uv; the reference's consumers split
        the CV_32FC2 result themselves, superres/src/optical_flow.cpp:557-574).  Returns (u, v)."""
        torch = _torch()
        if (u is None or v is None) and self._needs_initial_flow():
            raise B2FError(1)
        if u is None:
            u = torch.empty((I0.shape[0], I0.shape[1]), dtype=torch.float32, device=I0.device)
        if v is None:
            v = torch.empty_like(u)
        i0, i1 = _image_from_tensor(I0), _image_from_tensor(I1)
        iu, iv = _image_from_tensor(u), _image_from_tensor(v)
        if stream is None:
            stream = torch.cuda.current_stream(I0.device)
        sptr = stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)
        st = self._lib.b2f_calc_uv(self._h, C.byref(i0), C.byref(i1), C.byref(iu), C.byref(iv), C.c_void_p(sptr))
        if st != 0:
            raise B2FError(st, self._lib.b2f_last_cuda_error(self._h))
        return u, v

    def calc_host(self, I0: np.ndarray, I1: np.ndarray, flow: np.ndarray | None = None, stream=None):
        """Host-buffer variant (upload + calc + download inside the call; b2f_calc_host)."""
        if flow is None and self._needs_initial_flow():
            raise B2FError(1)
        if flow is None:
            flow = np.zeros((I0.shape[0], I0.shape[1], 2), np.float32)
        i0, i1, fl = _image_from_numpy(I0), _image_from_numpy(I1), _image_from_numpy(flow, True)
        sptr = 0
        if stream is not None:
            sptr = stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)
        else:
            sptr = _torch().cuda.current_stream().cuda_stream
        st = self._lib.b2f_calc_host(self._h, C.byref(i0), C.byref(i1), C.byref(fl), C.c_void_p(sptr))
        if st != 0:
            raise B2FError(st, self._lib.b2f_last_cuda_error(self._h))
        return flow

    # -- engine knobs / diagnostics (no reference counterpart)
    def _set(self, pid: int, v):
        st = self._lib.b2f_set_param(self._h, pid, float(v))
        if st != 0:
            raise B2FError(st)

    def _get(self, pid: int) -> float:
        out = C.c_double()
        st = self._lib.b2f_get_param(self._h, pid, C.byref(out))
        if st != 0:
            raise B2FError(st)
        return out.value

    def setEngineOption(self, name: str, v):
        self._set(PARAM["engine"][name], v)

    def getEngineOption(self, name: str) -> float:
        return self._get(PARAM["engine"][name])

    def setProfiling(self, on: bool):
        self._lib.b2f_set_profiling(self._h, int(on))

    def resetStats(self):
        self._lib.b2f_reset_stats(self._h)

    def getStats(self) -> dict:
        s = b2f_stats()
        self._lib.b2f_get_stats(self._h, C.byref(s))
        classes = {}
        for i in range(_lib.B2F_MAX_KERNEL_CLASSES):
            if s.class_launches[i]:
                classes[self._lib.b2f_kernel_class_name(self._h, i).decode()] = {
                    "launches": int(s.class_launches[i]), "ms": float(s.class_ms[i]),
                    "bytes": float(s.class_bytes[i])}
        return {"calls": int(s.calls), "launches": int(s.launches), "levels": int(s.levels),
                "iterations_run": int(s.iterations_run), "classes": classes}

    def workspaceBytes(self, rows: int = 0, cols: int = 0, type_: int = B2F_8UC1) -> int:
        return int(self._lib.b2f_workspace_bytes(self._h, rows, cols, type_))


def _accessors(cls, family: str, table):
    """Attach getX/setX pairs named as in cudaoptflow.hpp."""
    for pname, (camel, conv) in table.items():
        pid = PARAM[family][pname]

        def getter(self, _pid=pid, _conv=conv):
            return _conv(self._get(_pid))

        def setter(self, v, _pid=pid):
            self._set(_pid, v)

        setattr(cls, "get" + camel, getter)
        setattr(cls, "set" + camel, setter)


class OpticalFlowDual_TVL1(DenseOpticalFlow):
    """cv::cuda::OpticalFlowDual_TVL1 (cudaoptflow.hpp:305-386)."""

    def _needs_initial_flow(self) -> bool:
        return bool(self.getUseInitialFlow()) and self.getInitialFlowSource() == 0

    def getActivePath(self, level: int = 0) -> int:
        """What the last calc ran on pyramid level `level`: an OR of _lib.TVL1_PATH flags (B2F_ENGINE_ACTIVE_PATH)."""
        return int(self._get(PARAM["engine"]["active_path"] + level))


_accessors(OpticalFlowDual_TVL1, "tvl1", {
    "tau": ("Tau", float), "lambda_": ("Lambda", float), "theta": ("Theta", float),
    "nscales": ("NumScales", int), "warps": ("NumWarps", int), "epsilon": ("Epsilon", float),
    "iterations": ("NumIterations", int), "scale_step": ("ScaleStep", float), "gamma": ("Gamma", float),
    "use_initial_flow": ("UseInitialFlow", bool),
    # knobs of the reference's CPU / OpenCL class (cv::optflow::DualTVL1OpticalFlow), see include/b200flow.h
    "median_filtering": ("MedianFiltering", int), "median_period": ("MedianPeriod", int),
    "initial_flow_source": ("InitialFlowSource", int)})


class FarnebackOpticalFlow(DenseOpticalFlow):
    """cv::cuda::FarnebackOpticalFlow (cudaoptflow.hpp:258-294)."""

    def _needs_initial_flow(self) -> bool:
        return (int(self.getFlags()) & OPTFLOW_USE_INITIAL_FLOW) != 0

    def getActivePath(self, level: int = 0) -> int:
        """The fused iteration kernel the last calc ran on pyramid level `level`: a _lib.FARN_PATH value
        (B2F_ENGINE_ACTIVE_PATH)."""
        return int(self._get(PARAM["engine"]["active_path"] + level))


_accessors(FarnebackOpticalFlow, "farneback", {
    "num_levels": ("NumLevels", int), "pyr_scale": ("PyrScale", float), "fast_pyramids": ("FastPyramids", bool),
    "win_size": ("WinSize", int), "num_iters": ("NumIters", int), "poly_n": ("PolyN", int),
    "poly_sigma": ("PolySigma", float), "flags": ("Flags", int)})


class BroxOpticalFlow(DenseOpticalFlow):
    """cv::cuda::BroxOpticalFlow (cudaoptflow.hpp:155-186)."""

    def getActivePath(self, level: int):
        """The solver the last calc ran on pyramid level `level`: (a _lib.BROX_PATH value, solver iterations the first
        launch of each inner step ran) (B2F_ENGINE_ACTIVE_PATH)."""
        v = int(self._get(PARAM["engine"]["active_path"] + level))
        return v & 0xFF, (v >> 8) & 0xFF


_accessors(BroxOpticalFlow, "brox", {
    "alpha": ("FlowSmoothness", float), "gamma": ("GradientConstancyImportance", float),
    "scale_factor": ("PyramidScaleFactor", float), "inner_iterations": ("InnerIterations", int),
    "outer_iterations": ("OuterIterations", int), "solver_iterations": ("SolverIterations", int)})


class DensePyrLKOpticalFlow(DenseOpticalFlow):
    """cv::cuda::DensePyrLKOpticalFlow (cudaoptflow.hpp:230-250)."""

    def getWinSize(self):
        return (int(self._get(PARAM["denselk"]["win_width"])), int(self._get(PARAM["denselk"]["win_height"])))

    def setWinSize(self, sz):
        self._set(PARAM["denselk"]["win_width"], sz[0])
        self._set(PARAM["denselk"]["win_height"], sz[1])


_accessors(DensePyrLKOpticalFlow, "denselk", {
    "max_level": ("MaxLevel", int), "iters": ("NumIters", int), "use_initial_flow": ("UseInitialFlow", bool)})


def _create(cls, fn_name: str, params):
    l = _lib.lib()
    h = C.c_void_p()
    st = getattr(l, fn_name)(C.byref(params), C.byref(h))
    if st != 0:
        raise B2FError(st)
    return cls(h)


def OpticalFlowDual_TVL1_create(tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01,
                                iterations=300, scaleStep=0.8, gamma=0.0, useInitialFlow=False):
    """cv::cuda::OpticalFlowDual_TVL1::create (cudaoptflow.hpp:375-385)."""
    p = _lib.b2f_tvl1_params(tau, lambda_, theta, nscales, warps, epsilon, iterations, scaleStep, gamma,
                             int(useInitialFlow))
    return _create(OpticalFlowDual_TVL1, "b2f_tvl1_create", p)


def FarnebackOpticalFlow_create(numLevels=5, pyrScale=0.5, fastPyramids=False, winSize=13, numIters=10,
                                polyN=5, polySigma=1.1, flags=0):
    """cv::cuda::FarnebackOpticalFlow::create (cudaoptflow.hpp:285-293)."""
    p = _lib.b2f_farneback_params(numLevels, pyrScale, int(fastPyramids), winSize, numIters, polyN, polySigma,
                                  flags)
    return _create(FarnebackOpticalFlow, "b2f_farneback_create", p)


def BroxOpticalFlow_create(alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=5,
                           outer_iterations=150, solver_iterations=10):
    """cv::cuda::BroxOpticalFlow::create (cudaoptflow.hpp:179-185)."""
    p = _lib.b2f_brox_params(alpha, gamma, scale_factor, inner_iterations, outer_iterations, solver_iterations)
    return _create(BroxOpticalFlow, "b2f_brox_create", p)


def DensePyrLKOpticalFlow_create(winSize=(13, 13), maxLevel=3, iters=30, useInitialFlow=False):
    """cv::cuda::DensePyrLKOpticalFlow::create (cudaoptflow.hpp:245-249)."""
    p = _lib.b2f_denselk_params(winSize[0], winSize[1], maxLevel, iters, int(useInitialFlow))
    return _create(DensePyrLKOpticalFlow, "b2f_denselk_create", p)


def _sparse_image(t) -> b2f_image:
    """(H, W) or (H, W, C) CUDA tensor, C in {1, 3, 4}, dtype uint8 / uint16 / int32 / float32 -> b2f_image with OpenCV's
    CV_MAKETYPE(depth, C) flag: the instantiations of the reference's sparse dispatcher table (pyrlk.cpp:195-203)."""
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("expected a CUDA torch.Tensor (the GpuMat stand-in)")
    depth = {torch.uint8: 0, torch.uint16: 2, torch.int32: 4, torch.float32: 5}.get(t.dtype)
    if depth is None or t.dim() not in (2, 3):
        raise B2FError(2)
    cn = 1 if t.dim() == 2 else int(t.shape[2])
    if cn not in (1, 3, 4):
        raise B2FError(2)  # CV_Assert(channels == 1 || 3 || 4), pyrlk.cpp:228
    if t.dim() == 3 and (t.stride(2) != 1 or t.stride(1) != cn):
        raise ValueError("pixels must be interleaved and contiguous")
    if t.dim() == 2 and t.stride(1) != 1:
        raise ValueError("image rows must be contiguous")
    return b2f_image(t.data_ptr(), t.stride(0) * t.element_size(), t.shape[0], t.shape[1], depth + ((cn - 1) << 3))


class SparsePyrLKOpticalFlow:
    """cv::cuda::SparsePyrLKOpticalFlow (cudaoptflow.hpp:189-226).

        nextPts, status, err = alg.calc(prevImg, nextImg, prevPts[, nextPts[, status[, err[, stream]]]])

    prevPts / nextPts: CUDA float32 tensors of shape (1, N, 2) or (N, 2) (the reference's 1 x N CV_32FC2 GpuMat),
    status: uint8 (N,), err: float32 (N,) -- computed only when ``err`` is passed or ``wantErr=True``.
    """

    def __init__(self, handle):
        self._h = handle
        self._lib = _lib.lib()

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b2f_sparselk_destroy(h)

    def _params(self):
        p = _lib.b2f_sparselk_params()
        self._lib.b2f_sparselk_get_params(self._h, C.byref(p))
        return p

    def _update(self, **kw):
        p = self._params()
        for k, v in kw.items():
            setattr(p, k, int(v))
        self._lib.b2f_sparselk_set_params(self._h, C.byref(p))

    def getWinSize(self):
        p = self._params()
        return (p.win_width, p.win_height)

    def setWinSize(self, sz):
        self._update(win_width=sz[0], win_height=sz[1])

    def getMaxLevel(self):
        return self._params().max_level

    def setMaxLevel(self, v):
        self._update(max_level=v)

    def getNumIters(self):
        return self._params().iters

    def setNumIters(self, v):
        self._update(iters=v)

    def getUseInitialFlow(self):
        return bool(self._params().use_initial_flow)

    def setUseInitialFlow(self, v):
        self._update(use_initial_flow=bool(v))

    def getDefaultName(self) -> str:
        return "SparseOpticalFlow.SparsePyrLKOpticalFlow"

    def calc(self, prevImg, nextImg, prevPts, nextPts=None, status=None, err=None, stream=None, wantErr=False):
        torch = _torch()
        if prevPts.dtype != torch.float32 or prevPts.shape[-1] != 2 or not prevPts.is_contiguous():
            raise B2FError(2)  # CV_Assert(prevPts.rows == 1 && prevPts.type() == CV_32FC2), pyrlk.cpp:159
        n = prevPts.numel() // 2
        if nextPts is None:
            if self.getUseInitialFlow():
                raise B2FError(1)  # CV_Assert(nextPts.size() == prevPts.size()), pyrlk.cpp:162-163
            nextPts = torch.empty_like(prevPts)
        elif nextPts.shape != prevPts.shape or nextPts.dtype != torch.float32 or not nextPts.is_contiguous():
            raise B2FError(3)
        if status is None:
            status = torch.empty((n,), dtype=torch.uint8, device=prevPts.device)
        if err is None and wantErr:
            err = torch.empty((n,), dtype=torch.float32, device=prevPts.device)
        i0, i1 = _sparse_image(prevImg), _sparse_image(nextImg)
        if stream is None:
            stream = torch.cuda.current_stream(prevImg.device)
        sptr = stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)
        st = self._lib.b2f_sparselk_calc(self._h, C.byref(i0), C.byref(i1), C.c_void_p(prevPts.data_ptr()),
                                         C.c_void_p(nextPts.data_ptr()), C.c_void_p(status.data_ptr()),
                                         C.c_void_p(err.data_ptr()) if err is not None else None, n, C.c_void_p(sptr))
        if st != 0:
            raise B2FError(st)
        return nextPts, status, err


def SparsePyrLKOpticalFlow_create(winSize=(21, 21), maxLevel=3, iters=30, useInitialFlow=False):
    """cv::cuda::SparsePyrLKOpticalFlow::create (cudaoptflow.hpp:221-225)."""
    p = _lib.b2f_sparselk_params(winSize[0], winSize[1], maxLevel, iters, int(useInitialFlow))
    l = _lib.lib()
    h = C.c_void_p()
    st = l.b2f_sparselk_create(C.byref(p), C.byref(h))
    if st != 0:
        raise B2FError(st)
    return SparsePyrLKOpticalFlow(h)
