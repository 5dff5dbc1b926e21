"""cudaimgproc's corner classes (modules/cudaimgproc/include/opencv2/cudaimgproc.hpp:538-620), as the reference's
generated Python bindings expose them:

    crit = cv2.cuda.createMinEigenValCorner(srcType, blockSize, ksize[, borderType])
    dst = crit.compute(src[, dst[, stream]])                       # GpuMat CV_32FC1 out
    det = cv2.cuda.createGoodFeaturesToTrackDetector(srcType[, maxCorners[, qualityLevel[, minDistance[, ...]]]])
    corners = det.detect(image[, mask[, stream]])                  # 1 x N CV_32FC2

A GpuMat is a CUDA torch.Tensor and a Stream a torch.cuda.Stream, as in cudaoptflow.py.  ``detect`` returns a
(1, N, 2) float32 CUDA tensor, directly usable as SparsePyrLKOpticalFlow.calc's prevPts (empty, 1 x 0, when there is no
candidate).  Reading N is its one host read.
"""
from __future__ import annotations

import ctypes as C

from . import _lib
from ._lib import B2F_8UC1, B2F_32FC1, B2FError
from .cudaoptflow import _image_from_tensor, _torch
from .superres import _stream_ptr

BORDER_REPLICATE, BORDER_REFLECT, BORDER_REFLECT101 = 1, 2, 4


class _Handle:
    def __init__(self, handle):
        self._h = handle
        self._lib = _lib.lib()

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b2f_corners_destroy(h)

    def _check(self, st):
        if st != 0:
            raise B2FError(st, self._lib.b2f_corners_last_cuda_error(self._h))


class CornernessCriteria(_Handle):
    """cv::cuda::CornernessCriteria (cudaimgproc.hpp:538-567)."""

    def compute(self, src, dst=None, stream=None):
        torch = _torch()
        i = _image_from_tensor(src)
        if dst is None:
            dst = torch.empty(src.shape, dtype=torch.float32, device=src.device)
        o = _image_from_tensor(dst)
        self._check(self._lib.b2f_corners_compute(self._h, C.byref(i), C.byref(o), C.c_void_p(_stream_ptr(stream, src.device))))
        return dst


class CornersDetector(_Handle):
    """cv::cuda::CornersDetector (cudaimgproc.hpp:581-600), the GoodFeaturesToTrack detector."""

    def _params(self):
        p = _lib.b2f_gftt_params()
        self._check(self._lib.b2f_gftt_get_params(self._h, C.byref(p)))
        return p

    def setMaxCorners(self, maxCorners):
        p = self._params()
        p.max_corners = int(maxCorners)
        self._check(self._lib.b2f_gftt_set_params(self._h, C.byref(p)))

    def setMinDistance(self, minDistance):
        p = self._params()
        p.min_distance = float(minDistance)
        self._check(self._lib.b2f_gftt_set_params(self._h, C.byref(p)))

    def capacity(self, rows, cols) -> int:
        n = C.c_int()
        self._check(self._lib.b2f_gftt_capacity(self._h, rows, cols, C.byref(n)))
        return n.value

    def detect_async(self, image, mask=None, corners=None, count=None, stream=None):
        """The device-only form: fills ``corners`` ((capacity, 2) float32) and ``count`` (int32, 1) on the stream and
        returns them without any host read."""
        torch = _torch()
        img = _image_from_tensor(image)
        m = _image_from_tensor(mask) if mask is not None else None
        cap = self.capacity(image.shape[0], image.shape[1])
        if corners is None:
            corners = torch.empty((cap, 2), dtype=torch.float32, device=image.device)
        if count is None:
            count = torch.empty((1,), dtype=torch.int32, device=image.device)
        if corners.dtype != torch.float32 or not corners.is_contiguous() or corners.numel() < 2 * cap:
            raise B2FError(1)
        if count.dtype != torch.int32:
            raise B2FError(1)
        self._check(self._lib.b2f_gftt_detect(self._h, C.byref(img), C.byref(m) if m is not None else None,
                                              C.c_void_p(corners.data_ptr()), corners.numel() // 2,
                                              C.c_void_p(count.data_ptr()), C.c_void_p(_stream_ptr(stream, image.device))))
        return corners, count

    def detect(self, image, mask=None, stream=None):
        corners, count = self.detect_async(image, mask, stream=stream)
        torch = _torch()
        if stream is not None:
            s = stream if isinstance(stream, torch.cuda.Stream) else torch.cuda.ExternalStream(int(stream))
            with torch.cuda.stream(s):
                n = int(count.item())
        else:
            n = int(count.item())
        return corners[:n].view(1, n, 2)

    def lastInfo(self, stream=None) -> dict:
        """What the last detect did: candidates found, kept after the capacity cut, whether the cut applied, and the
        rounds of the minDistance selection.  Waits for the stream."""
        info = _lib.b2f_gftt_info()
        torch = _torch()
        self._check(self._lib.b2f_gftt_last_info(self._h, C.byref(info), C.c_void_p(_stream_ptr(stream, torch.cuda.current_device()))))
        return dict(candidates=info.candidates, kept=info.kept, capped=bool(info.capped), rounds=info.rounds)


def _src_type(srcType):
    if srcType not in (B2F_8UC1, B2F_32FC1):
        raise B2FError(2)
    return srcType


def createHarrisCorner(srcType, blockSize, ksize, k, borderType=BORDER_REFLECT101):
    """cv::cuda::createHarrisCorner (cudaimgproc.hpp:569-575)."""
    l = _lib.lib()
    h = C.c_void_p()
    st = l.b2f_harris_create(_src_type(srcType), blockSize, ksize, float(k), borderType, C.byref(h))
    if st != 0:
        raise B2FError(st)
    return CornernessCriteria(h)


def createMinEigenValCorner(srcType, blockSize, ksize, borderType=BORDER_REFLECT101):
    """cv::cuda::createMinEigenValCorner (cudaimgproc.hpp:577-579)."""
    l = _lib.lib()
    h = C.c_void_p()
    st = l.b2f_mineig_create(_src_type(srcType), blockSize, ksize, borderType, C.byref(h))
    if st != 0:
        raise B2FError(st)
    return CornernessCriteria(h)


def createGoodFeaturesToTrackDetector(srcType, maxCorners=1000, qualityLevel=0.01, minDistance=0.0, blockSize=3,
                                      useHarrisDetector=False, harrisK=0.04):
    """cv::cuda::createGoodFeaturesToTrackDetector (cudaimgproc.hpp:610-620)."""
    l = _lib.lib()
    p = _lib.b2f_gftt_params(int(maxCorners), float(qualityLevel), float(minDistance), int(blockSize),
                             int(bool(useHarrisDetector)), float(harrisK))
    h = C.c_void_p()
    st = l.b2f_gftt_create(_src_type(srcType), C.byref(p), C.byref(h))
    if st != 0:
        raise B2FError(st)
    return CornersDetector(h)
