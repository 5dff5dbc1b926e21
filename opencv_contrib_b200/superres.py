"""Python mirror of the reference's superres module on the GPU (modules/superres/include/opencv2/superres.hpp,
superres/optical_flow.hpp): BTV-L1 video super-resolution and its four CUDA optical-flow wrappers.

    sr = createSuperResolution_BTVL1_CUDA()
    sr.setInput(frames)                  # an object with nextFrame() [and reset()], or an iterable of frames
    while (out := sr.nextFrame()) is not None:
        ...                              # H s - 2 btv x W s - 2 btv [x C] uint8 CUDA tensor

Frames are H x W[ x C] uint8 (C = 3 or 4 is BGR / BGRA), numpy arrays or CUDA tensors.  The pull schedule runs in
libb200flow.so (b2f_superres_*); this module only feeds it frames.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import B2FError, b2f_image, b2f_stats
from .cudaoptflow import (BroxOpticalFlow_create, DensePyrLKOpticalFlow_create, FarnebackOpticalFlow_create,
                          OpticalFlowDual_TVL1_create, _torch)

_U8_TYPES = {1: 0, 3: 16, 4: 24}
_F32_TYPES = {1: 5, 3: 21, 4: 29}


def _stream_ptr(stream, device):
    torch = _torch()
    if stream is None:
        stream = torch.cuda.current_stream(device)
    return stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)


def _frame_tensor(f):
    torch = _torch()
    if isinstance(f, np.ndarray):
        f = torch.from_numpy(np.ascontiguousarray(f)).cuda()
    if not isinstance(f, torch.Tensor) or not f.is_cuda:
        raise TypeError("frames are uint8 numpy arrays or CUDA tensors")
    if f.dtype != torch.uint8 or f.dim() not in (2, 3) or (f.dim() == 3 and f.shape[2] not in (1, 3, 4)):
        raise B2FError(2)
    return f.contiguous()


def _image(t) -> b2f_image:
    cn = 1 if t.dim() == 2 else int(t.shape[2])
    table = _U8_TYPES if t.element_size() == 1 else _F32_TYPES
    return b2f_image(t.data_ptr(), t.stride(0) * t.element_size(), t.shape[0], t.shape[1], table[cn])


class DenseOpticalFlowExt:
    """cv::superres::DenseOpticalFlowExt over one of the cudaoptflow engines (superres/src/optical_flow.cpp:440-849):
    calc(frame0, frame1, flow1=None, flow2=None) converts the frames to the engine's work type (BGR(A) -> gray, then
    8UC1, or 32FC1 in [0, 1] for Brox) and returns the interleaved flow, or (u, v) when flow2 is requested (pass
    flow2=True to have it allocated)."""

    _table: dict = {}

    def __init__(self, engine):
        self._engine = engine

    @property
    def _h(self):
        return self._engine._h

    def calc(self, frame0, frame1, flow1=None, flow2=None, stream=None):
        torch = _torch()
        f0, f1 = _frame_tensor(frame0), _frame_tensor(frame1)
        h, w = f0.shape[:2]
        l = _lib.lib()
        sptr = _stream_ptr(stream, f0.device)
        if flow2 is not None:
            u = flow1 if flow1 is not None else torch.empty((h, w), dtype=torch.float32, device=f0.device)
            v = flow2 if not isinstance(flow2, bool) else torch.empty((h, w), dtype=torch.float32, device=f0.device)
            st = l.b2f_calc_ext(self._h, C.byref(_image(f0)), C.byref(_image(f1)), C.byref(_image(u)),
                                C.byref(_image(v)), C.c_void_p(sptr))
            if st != 0:
                raise B2FError(st, l.b2f_last_cuda_error(self._h))
            return u, v
        flow = flow1 if flow1 is not None else torch.empty((h, w, 2), dtype=torch.float32, device=f0.device)
        fl = b2f_image(flow.data_ptr(), flow.stride(0) * 4, h, w, _lib.B2F_32FC2)
        st = l.b2f_calc_ext(self._h, C.byref(_image(f0)), C.byref(_image(f1)), C.byref(fl), None, C.c_void_p(sptr))
        if st != 0:
            raise B2FError(st, l.b2f_last_cuda_error(self._h))
        return flow

    def collectGarbage(self):
        pass

    def __getattr__(self, name):
        # the superres getter / setter names, mapped onto the engine's
        table = type(self)._table
        if name[:3] in ("get", "set") and name[3:] in table:
            target = getattr(self._engine, name[:3] + table[name[3:]])
            return target
        raise AttributeError(name)


class FarnebackOpticalFlow(DenseOpticalFlowExt):
    _table = {"PyrScale": "PyrScale", "LevelsNumber": "NumLevels", "WindowSize": "WinSize", "Iterations": "NumIters",
              "PolyN": "PolyN", "PolySigma": "PolySigma", "Flags": "Flags"}


class DualTVL1OpticalFlow(DenseOpticalFlowExt):
    _table = {"Tau": "Tau", "Lambda": "Lambda", "Theta": "Theta", "ScalesNumber": "NumScales",
              "WarpingsNumber": "NumWarps", "Epsilon": "Epsilon", "Iterations": "NumIterations",
              "UseInitialFlow": "UseInitialFlow"}


class BroxOpticalFlow(DenseOpticalFlowExt):
    _table = {"Alpha": "FlowSmoothness", "Gamma": "GradientConstancyImportance", "ScaleFactor": "PyramidScaleFactor",
              "InnerIterations": "InnerIterations", "OuterIterations": "OuterIterations",
              "SolverIterations": "SolverIterations"}


class PyrLKOpticalFlow(DenseOpticalFlowExt):
    _table = {"MaxLevel": "MaxLevel", "Iterations": "NumIters"}

    def getWindowSize(self):
        return self._engine.getWinSize()[0]

    def setWindowSize(self, v):
        self._engine.setWinSize((v, v))


def createOptFlow_Farneback_CUDA():
    return FarnebackOpticalFlow(FarnebackOpticalFlow_create())


def createOptFlow_DualTVL1_CUDA():
    return DualTVL1OpticalFlow(OpticalFlowDual_TVL1_create())


def createOptFlow_Brox_CUDA():
    """Brox_CUDA's engine: cuda::BroxOpticalFlow::create(0.197f, 50.0f, 0.8f, 10, 77, 10) (optical_flow.cpp:533)."""
    f = lambda x: float(np.float32(x))
    return BroxOpticalFlow(BroxOpticalFlow_create(f(0.197), f(50.0), f(0.8), 10, 77, 10))


def createOptFlow_PyrLK_CUDA():
    return PyrLKOpticalFlow(DensePyrLKOpticalFlow_create())


_P = _lib.PARAM["superres"]
_SR_PARAMS = {"Scale": (_P["scale"], int), "Iterations": (_P["iterations"], int), "Tau": (_P["tau"], float),
              "Lambda": (_P["lambda_"], float), "Alpha": (_P["alpha"], float), "KernelSize": (_P["btv_kernel_size"], int),
              "BlurKernelSize": (_P["blur_kernel_size"], int), "BlurSigma": (_P["blur_sigma"], float),
              "TemporalAreaRadius": (_P["temporal_area_radius"], int)}


class _IterSource:
    def __init__(self, it):
        self._items = it
        self._it = iter(it)

    def nextFrame(self):
        return next(self._it, None)

    def reset(self):
        self._it = iter(self._items)


class SuperResolution:
    """cv::superres::SuperResolution as createSuperResolution_BTVL1_CUDA builds it (superres.hpp:68-190)."""

    def __init__(self):
        self._lib = _lib.lib()
        self._flow = createOptFlow_Farneback_CUDA()
        h = C.c_void_p()
        st = self._lib.b2f_superres_create(None, self._flow._h, C.byref(h))
        if st != 0:
            raise B2FError(st)
        self._sr = h
        self._source = None

    def __del__(self):
        h, self._sr = getattr(self, "_sr", None), None
        if h:
            self._lib.b2f_superres_destroy(h)

    def _check(self, st):
        if st != 0:
            raise B2FError(st, self._lib.b2f_superres_last_cuda_error(self._sr))

    # -- parameters
    def _set(self, pid, v):
        self._check(self._lib.b2f_superres_set_param(self._sr, pid, float(v)))

    def _get(self, pid):
        out = C.c_double()
        self._check(self._lib.b2f_superres_get_param(self._sr, pid, C.byref(out)))
        return out.value

    def getOpticalFlow(self):
        return self._flow

    def setOpticalFlow(self, flow):
        """One of the createOptFlow_*_CUDA wrappers, or any object with calc(frame0, frame1, flow1, flow2) that returns
        (or fills) the planar flow -- such an object runs through the caller-supplied-flow path."""
        self._flow = flow
        self._check(self._lib.b2f_superres_set_flow(self._sr, flow._h if isinstance(flow, DenseOpticalFlowExt) else None))

    def setEngineOption(self, name, v):
        self._set(_lib.PARAM["engine"][name], v)

    # -- frame source
    def setInput(self, source):
        if not hasattr(source, "nextFrame"):
            source = _IterSource(list(source) if not isinstance(source, (list, tuple)) else source)
        self._source = source
        self._prev = None
        self._check(self._lib.b2f_superres_reset(self._sr))

    def reset(self):
        if self._source is not None and hasattr(self._source, "reset"):
            self._source.reset()
        self._prev = None
        self._check(self._lib.b2f_superres_reset(self._sr))

    def collectGarbage(self):
        self._prev = None
        self._check(self._lib.b2f_superres_collect_garbage(self._sr))

    def _push(self, frame, sptr):
        l = self._lib
        if frame is None or (hasattr(frame, "numel") and frame.numel() == 0) or (
                isinstance(frame, np.ndarray) and frame.size == 0):
            if isinstance(self._flow, DenseOpticalFlowExt):
                return self._check(l.b2f_superres_push(self._sr, None, C.c_void_p(sptr)))
            return self._check(l.b2f_superres_push_flows(self._sr, None, None, None, None, None, C.c_void_p(sptr)))
        t = _frame_tensor(frame)
        self._cn = 1 if t.dim() == 2 else int(t.shape[2])
        if isinstance(self._flow, DenseOpticalFlowExt):
            return self._check(l.b2f_superres_push(self._sr, C.byref(_image(t)), C.c_void_p(sptr)))
        torch = _torch()
        imgs, flows = [None] * 4, []  # the flows stay referenced until the push has read them
        prev = getattr(self, "_prev", None)
        if prev is not None:
            h, w = t.shape[:2]
            for a, b in ((prev, t), (t, prev)):
                u = torch.zeros((h, w), dtype=torch.float32, device=t.device)
                v = torch.zeros_like(u)
                r = self._flow.calc(a, b, u, v)
                if isinstance(r, tuple) and len(r) == 2:
                    u, v = (x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x, np.float32)).to(t.device)
                            for x in r)
                flows += [u.float().contiguous(), v.float().contiguous()]
            imgs = [C.pointer(_image(f)) for f in flows]
        st = l.b2f_superres_push_flows(self._sr, C.byref(_image(t)), *imgs, C.c_void_p(sptr))
        self._check(st)
        self._prev = t

    def nextFrame(self, float_output=False, stream=None):
        """The next output frame (uint8, or the float estimate before convertTo with float_output=True), None at the
        end of the stream."""
        torch = _torch()
        l = self._lib
        sptr = _stream_ptr(stream, torch.device("cuda", torch.cuda.current_device()))
        wants = C.c_int()
        while True:
            self._check(l.b2f_superres_wants_frame(self._sr, C.byref(wants)))
            if not wants.value:
                break
            self._push(self._source.nextFrame(), sptr)
        rows, cols = C.c_int(), C.c_int()
        if l.b2f_superres_output_size(self._sr, C.byref(rows), C.byref(cols)) != 0:
            rows.value = cols.value = 1  # no frame in the stream: the pop reports the end
        cn = getattr(self, "_cn", 1)
        shape = (rows.value, cols.value) if cn == 1 else (rows.value, cols.value, cn)
        out = torch.empty(shape, dtype=torch.float32 if float_output else torch.uint8, device="cuda")
        got = C.c_int()
        self._check(l.b2f_superres_pop(self._sr, C.byref(_image(out)), C.byref(got), C.c_void_p(sptr)))
        return out if got.value else None

    def getStats(self):
        s = b2f_stats()
        self._lib.b2f_superres_get_stats(self._sr, C.byref(s))
        return {"launches": int(s.launches), "calls": int(s.calls), "iterations_run": int(s.iterations_run)}

    def resetStats(self):
        self._lib.b2f_superres_reset_stats(self._sr)


def _accessors():
    for camel, (pid, conv) in _SR_PARAMS.items():
        setattr(SuperResolution, "get" + camel, lambda self, _p=pid, _c=conv: _c(self._get(_p)))
        setattr(SuperResolution, "set" + camel, lambda self, v, _p=pid: self._set(_p, v))


_accessors()


def createSuperResolution_BTVL1_CUDA():
    """cv::superres::createSuperResolution_BTVL1_CUDA (btv_l1_cuda.cpp:584-587): Farneback flows by default."""
    return SuperResolution()
