"""The video module's pyramidal Lucas-Kanade tracker (video/tracking.hpp) on the GPU, with cv2's names and semantics:

    retval, pyramid = buildOpticalFlowPyramid(img, winSize, maxLevel[, pyramid[, withDerivatives[, pyrBorder[,
                                              derivBorder[, tryReuseInputImage[, stream]]]]]])
    nextPts, status, err = calcOpticalFlowPyrLK(prevImg, nextImg, prevPts, nextPts[, status[, err[, winSize[,
                                                maxLevel[, criteria[, flags[, minEigThreshold[, stream]]]]]]]])
    lk = SparsePyrLKOpticalFlow_create(winSize, maxLevel, crit, flags, minEigThreshold)
    nextPts, status, err = lk.calc(prevImg, nextImg, prevPts, nextPts[, status[, err[, stream]]])

Results equal cv2 4.13 bit for bit (DESIGN §4.13).  Frames are CUDA uint8 tensors (H, W) or (H, W, C), rows may be
pitched; prevImg / nextImg may each be an ``OpticalFlowPyramid`` instead, which is how a video loop reuses frame t+1's
pyramid as the next pair's prev.  Points are CUDA float32 tensors (1, N, 2), (N, 1, 2) or (N, 2), so
CornersDetector.detect's output goes straight in; status is (N, 1) uint8 and err (N, 1) float32, as cv2 returns them.
Everything runs on the stream (default: torch's current stream) without a host read.

This tracker follows the CPU video module.  ``opencv_contrib_b200.SparsePyrLKOpticalFlow_create`` is the cv::cuda one.
"""
from __future__ import annotations

import ctypes as C
import threading
import weakref

from . import _lib
from ._lib import B2FError
from .cudaoptflow import _torch
from .superres import _stream_ptr

OPTFLOW_USE_INITIAL_FLOW = 4
OPTFLOW_LK_GET_MIN_EIGENVALS = 8
BORDER_CONSTANT, BORDER_REFLECT_101, BORDER_ISOLATED = 0, 4, 16
TERM_CRITERIA_COUNT, TERM_CRITERIA_EPS = 1, 2


def _check(st, cuda_error=0):
    if st != 0:
        raise B2FError(st, cuda_error)


def _frame(t):
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError("expected a CUDA torch.Tensor or an OpticalFlowPyramid")
    if t.dtype != torch.uint8 or t.dim() not in (2, 3):
        raise B2FError(2)  # CV_Assert(depth == CV_8U)
    cn = 1 if t.dim() == 2 else t.shape[2]
    if (t.dim() == 3 and t.stride(2) != 1) or t.stride(1) != cn:
        raise ValueError("frame pixels must be contiguous and interleaved")
    if not 1 <= cn <= 256:
        raise B2FError(2)
    return _lib.b2f_image(t.data_ptr(), t.stride(0), t.shape[0], t.shape[1], (cn - 1) << 3)


class _DeviceView:
    """__cuda_array_interface__ over a pyramid level; keeps the pyramid alive while a tensor uses it."""

    def __init__(self, owner, ptr, shape, strides, typestr):
        self._owner = owner
        self.__cuda_array_interface__ = dict(shape=shape, strides=strides, typestr=typestr, data=(ptr, False),
                                             version=2)


class OpticalFlowPyramid:
    """A device pyramid as buildOpticalFlowPyramid makes it: uint8 levels with a winSize border and, optionally, int16
    Scharr derivatives (Ix, Iy per channel) with a zero border.

    The tensors padded(), level() and tolist() return view the pyramid's memory.  Rebuilding the pyramid in place at
    the same geometry refreshes what they show; a rebuild at another geometry (size, channels, window, level count or
    derivatives) would move the levels, so it is refused while such a view is alive."""

    def __init__(self):
        self._lib = _lib.lib()
        h = C.c_void_p()
        _check(self._lib.b2f_lkpyr_pyramid_create(C.byref(h)))
        self._h = h
        self.device = None
        self._geometry = None
        self._views = weakref.WeakSet()  # the _DeviceView objects live tensors hold

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b2f_lkpyr_pyramid_destroy(h)

    def info(self):
        lv, ww, wh, d = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _check(self._lib.b2f_lkpyr_pyramid_info(self._h, C.byref(lv), C.byref(ww), C.byref(wh), C.byref(d)))
        return dict(levels=lv.value, winSize=(ww.value, wh.value), withDerivatives=bool(d.value))

    def __len__(self):
        return self.info()["levels"]

    def padded(self, level, deriv=False):
        """Level `level` (or its derivatives) with its border, (rows + 2 wh, cols + 2 ww, C) -- a view, no copy."""
        torch = _torch()
        v = _lib.b2f_image()
        _check(self._lib.b2f_lkpyr_pyramid_level(self._h, level, int(bool(deriv)), C.byref(v)))
        cn = (v.type >> 3) + 1
        es = 2 if deriv else 1
        view = _DeviceView(self, v.data, (v.rows, v.cols, cn), (v.step, cn * es, es), "<i2" if deriv else "|u1")
        self._views.add(view)
        return torch.as_tensor(view, device=self.device)

    def level(self, level, deriv=False):
        """The level without its border, as cv2's returned list holds it."""
        ww, wh = self.info()["winSize"]
        p = self.padded(level, deriv)
        return p[wh:p.shape[0] - wh, ww:p.shape[1] - ww]

    def tolist(self):
        """cv2's list: [level 0, derivatives 0, level 1, ...] (derivatives only when built with them)."""
        inf = self.info()
        out = []
        for i in range(inf["levels"]):
            out.append(self.level(i))
            if inf["withDerivatives"]:
                out.append(self.level(i, True))
        return out


def buildOpticalFlowPyramid(img, winSize, maxLevel, pyramid=None, withDerivatives=True, pyrBorder=BORDER_REFLECT_101,
                            derivBorder=BORDER_CONSTANT, tryReuseInputImage=True, stream=None):
    """cv::buildOpticalFlowPyramid.  Returns (maxLevel built, OpticalFlowPyramid); a `pyramid` passed in is rebuilt in
    place (its memory reused when it is large enough).  Only BORDER_REFLECT_101 levels and BORDER_CONSTANT derivatives
    are built (other modes: B2F_UNSUPPORTED_TYPE).  The level-0 image is always copied into the padded level;
    tryReuseInputImage is accepted for cv2's signature."""
    del tryReuseInputImage
    l = _lib.lib()
    im = _frame(img)
    if pyramid is None:
        pyramid = OpticalFlowPyramid()
    geometry = (im.rows, im.cols, im.type, int(winSize[0]), int(winSize[1]),
                _levels(im.rows, im.cols, int(winSize[0]), int(winSize[1]), int(maxLevel)), bool(withDerivatives))
    if pyramid._geometry is not None and geometry != pyramid._geometry and len(pyramid._views):
        raise ValueError("the pyramid has live level views; rebuilding it at another geometry would move its levels")
    pyramid.device = img.device
    out = C.c_int()
    _check(l.b2f_lkpyr_build_pyramid(C.byref(im), int(winSize[0]), int(winSize[1]), int(maxLevel), int(bool(withDerivatives)),
                                     int(pyrBorder), int(derivBorder), pyramid._h, C.byref(out),
                                     C.c_void_p(_stream_ptr(stream, img.device))))
    pyramid._geometry = geometry
    return out.value, pyramid


def _levels(rows, cols, ww, wh, max_level):
    """buildOpticalFlowPyramid's return value for an image of rows x cols."""
    w, h = cols, rows
    for level in range(max(max_level, 0) + 1):
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= ww or h <= wh:
            return level
    return max_level


def _points(t):
    torch = _torch()
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
        raise TypeError("points are a CUDA float32 tensor")
    if not (t.dim() == 2 and t.shape[1] == 2) and not (t.dim() == 3 and 1 in t.shape[:2] and t.shape[2] == 2):
        raise B2FError(1)  # checkVector(2, CV_32F, true)
    if not t.is_contiguous():
        raise ValueError("points must be contiguous")
    return t.numel() // 2


class SparsePyrLKOpticalFlow:
    """cv::SparsePyrLKOpticalFlow (video/tracking.hpp), the class behind calcOpticalFlowPyrLK."""

    def __init__(self, handle):
        self._h = handle
        self._lib = _lib.lib()

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b2f_lkpyr_destroy(h)

    def _params(self):
        p = _lib.b2f_lkpyr_params()
        _check(self._lib.b2f_lkpyr_get_params(self._h, C.byref(p)))
        return p

    def _set(self, **kw):
        p = self._params()
        for k, v in kw.items():
            setattr(p, k, v)
        _check(self._lib.b2f_lkpyr_set_params(self._h, C.byref(p)))

    def getWinSize(self):
        p = self._params()
        return (p.win_width, p.win_height)

    def setWinSize(self, winSize):
        self._set(win_width=int(winSize[0]), win_height=int(winSize[1]))

    def getMaxLevel(self):
        return self._params().max_level

    def setMaxLevel(self, maxLevel):
        self._set(max_level=int(maxLevel))

    def getTermCriteria(self):
        p = self._params()
        return (p.criteria_type, p.max_count, p.epsilon)

    def setTermCriteria(self, crit):
        self._set(criteria_type=int(crit[0]), max_count=int(crit[1]), epsilon=float(crit[2]))

    def getFlags(self):
        return self._params().flags

    def setFlags(self, flags):
        self._set(flags=int(flags))

    def getMinEigThreshold(self):
        return self._params().min_eig_threshold

    def setMinEigThreshold(self, minEigThreshold):
        self._set(min_eig_threshold=float(minEigThreshold))

    def getDefaultName(self):
        return "SparsePyrLKOpticalFlow"

    def getActivePath(self):
        """What the last calc ran: bits 0-7 the tracker kernel (1: one thread per point, every level in one launch),
        bits 8-15 the levels it tracked."""
        v = C.c_double()
        eng = self._lib.b2f_lkpyr_engine(self._h)
        _check(self._lib.b2f_get_param(eng, _lib.PARAM["engine"]["active_path"], C.byref(v)))
        return int(v.value)

    def getStats(self):
        s = _lib.b2f_stats()
        _check(self._lib.b2f_get_stats(self._lib.b2f_lkpyr_engine(self._h), C.byref(s)))
        return dict(calls=s.calls, launches=s.launches)

    def calc(self, prevImg, nextImg, prevPts, nextPts=None, status=None, err=None, stream=None):
        torch = _torch()
        n = _points(prevPts)
        dev = prevPts.device
        flags = self._params().flags
        if nextPts is None:
            if flags & OPTFLOW_USE_INITIAL_FLOW:
                raise B2FError(1)  # cv2 asserts on nextPts' size
            nextPts = torch.empty_like(prevPts)
        if _points(nextPts) != n:
            raise B2FError(3)
        if status is None:
            status = torch.empty((n, 1), dtype=torch.uint8, device=dev)
        if err is None:
            err = torch.zeros((n, 1), dtype=torch.float32, device=dev)
        if status.dtype != torch.uint8 or status.numel() != n or not status.is_contiguous():
            raise B2FError(1)
        if err.dtype != torch.float32 or err.numel() != n or not err.is_contiguous():
            raise B2FError(1)
        args = []
        for f in (prevImg, nextImg):
            if isinstance(f, OpticalFlowPyramid):
                args += [None, f._h]
            else:
                args += [C.byref(_frame(f)), None]
        s = C.c_void_p(_stream_ptr(stream, dev))
        st = self._lib.b2f_lkpyr_calc(self._h, args[0], args[1], args[2], args[3], C.c_void_p(prevPts.data_ptr()),
                                      C.c_void_p(nextPts.data_ptr()), C.c_void_p(status.data_ptr()),
                                      C.c_void_p(err.data_ptr()), n, s)
        if st != 0:
            raise B2FError(st, self._lib.b2f_lkpyr_last_cuda_error(self._h))
        return nextPts, status, err


def SparsePyrLKOpticalFlow_create(winSize=(21, 21), maxLevel=3, crit=(TERM_CRITERIA_COUNT | TERM_CRITERIA_EPS, 30, 0.01),
                                  flags=0, minEigThreshold=1e-4):
    """cv::SparsePyrLKOpticalFlow::create."""
    l = _lib.lib()
    p = _lib.b2f_lkpyr_params(int(winSize[0]), int(winSize[1]), int(maxLevel), int(crit[0]), int(crit[1]), float(crit[2]),
                              int(flags), float(minEigThreshold))
    h = C.c_void_p()
    _check(l.b2f_lkpyr_create(C.byref(p), C.byref(h)))
    return SparsePyrLKOpticalFlow(h)


_handles = threading.local()


def calcOpticalFlowPyrLK(prevImg, nextImg, prevPts, nextPts=None, status=None, err=None, winSize=(21, 21), maxLevel=3,
                         criteria=(TERM_CRITERIA_COUNT | TERM_CRITERIA_EPS, 30, 0.01), flags=0, minEigThreshold=1e-4,
                         stream=None):
    """cv::calcOpticalFlowPyrLK, on a per-thread, per-device handle whose workspace persists between calls.  Calls on
    different streams are safe: the handle orders each call after the previous one when the stream changes."""
    cache = getattr(_handles, "d", None)
    if cache is None:
        cache = _handles.d = {}
    key = prevPts.device.index if hasattr(prevPts, "device") else None
    lk = cache.get(key)
    if lk is None:
        lk = cache[key] = SparsePyrLKOpticalFlow_create()
    lk._set(win_width=int(winSize[0]), win_height=int(winSize[1]), max_level=int(maxLevel), criteria_type=int(criteria[0]),
            max_count=int(criteria[1]), epsilon=float(criteria[2]), flags=int(flags),
            min_eig_threshold=float(minEigThreshold))
    return lk.calc(prevImg, nextImg, prevPts, nextPts, status, err, stream)
