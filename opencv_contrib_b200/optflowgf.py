"""The video module's Farneback flow (video/tracking.hpp) on the GPU, with cv2's names and semantics:

    flow = calcOpticalFlowFarneback(prev, next, flow, pyr_scale, levels, winsize, iterations, poly_n, poly_sigma,
                                    flags[, stream])
    fb = FarnebackOpticalFlow_create(numLevels, pyrScale, fastPyramids, winSize, numIters, polyN, polySigma, flags)
    flow = fb.calc(I0, I1, flow[, stream]);  fb.getPyrScale() / fb.setPyrScale(v) ...

Results equal cv2's portable CPU path (``cv2.setUseOptimized(False)`` with IPP off) bit for bit (DESIGN §4.14).  Frames
are CUDA uint8 or float32 tensors (H, W), rows may be pitched; the flow is a CUDA float32 (H, W, 2) tensor, read first
with OPTFLOW_USE_INITIAL_FLOW.  Everything runs on the stream (default: torch's current stream) without a host read.

``opencv_contrib_b200.FarnebackOpticalFlow`` is the cv::cuda class; this module's class follows the CPU one.
"""
from __future__ import annotations

import threading

from . import _lib
from .cudaoptflow import OPTFLOW_FARNEBACK_GAUSSIAN, OPTFLOW_USE_INITIAL_FLOW, DenseOpticalFlow, _accessors, _create

__all__ = ["FarnebackOpticalFlow", "FarnebackOpticalFlow_create", "calcOpticalFlowFarneback",
           "OPTFLOW_USE_INITIAL_FLOW", "OPTFLOW_FARNEBACK_GAUSSIAN", "PATH"]

# B2F_ENGINE_ACTIVE_PATH bits of this engine (include/b200flow.h)
PATH = dict(box=1, gaussian=2, area_level=4)


class FarnebackOpticalFlow(DenseOpticalFlow):
    """cv::FarnebackOpticalFlow (opencv's video module) on the GPU, with cv2's accessor names.  ``calc(I0, I1, flow)``
    returns the flow; with OPTFLOW_USE_INITIAL_FLOW in the flags the given flow is read first.  One handle may be
    called on several streams (a call on another stream waits for the previous call); for concurrent pairs use one
    handle per stream.  Its workspace holds 35 to 43 frame-size float planes (about 300 to 360 MB at 1080p, see
    workspaceBytes) and is kept until the handle is freed."""

    def _needs_initial_flow(self) -> bool:
        return (int(self.getFlags()) & OPTFLOW_USE_INITIAL_FLOW) != 0

    def getActivePath(self, level: int = 0) -> int:
        """What the last calc ran on pyramid level `level` (finest first): an OR of PATH bits."""
        return int(self._get(_lib.PARAM["engine"]["active_path"] + level))


_accessors(FarnebackOpticalFlow, "farneback", {
    "num_levels": ("NumLevels", int), "pyr_scale": ("PyrScale", float), "fast_pyramids": ("FastPyramids", bool),
    "win_size": ("WinSize", int), "num_iters": ("NumIters", int), "poly_n": ("PolyN", int),
    "poly_sigma": ("PolySigma", float), "flags": ("Flags", int)})


def FarnebackOpticalFlow_create(numLevels=5, pyrScale=0.5, fastPyramids=False, winSize=13, numIters=10, polyN=5,
                                polySigma=1.1, flags=0):
    """cv::FarnebackOpticalFlow::create (cv2.FarnebackOpticalFlow_create), with its defaults."""
    p = _lib.b2f_farneback_params(numLevels, pyrScale, int(fastPyramids), winSize, numIters, polyN, polySigma, flags)
    return _create(FarnebackOpticalFlow, "b2f_optflowgf_create", p)


_handles = threading.local()


def calcOpticalFlowFarneback(prev, next, flow, pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags,
                             stream=None):
    """cv::calcOpticalFlowFarneback with cv2's positional signature on CUDA tensors; returns the flow (a new tensor when
    ``flow`` is None).  One handle per host thread and device keeps its workspace and graph between calls; calls on
    different streams are safe, since the handle orders a call on another stream after the previous one."""
    cache = getattr(_handles, "d", None)
    if cache is None:
        cache = _handles.d = {}
    fb = cache.get(prev.device.index)
    if fb is None:
        fb = cache[prev.device.index] = FarnebackOpticalFlow_create()
    fb.setPyrScale(pyr_scale)
    fb.setNumLevels(levels)
    fb.setWinSize(winsize)
    fb.setNumIters(iterations)
    fb.setPolyN(poly_n)
    fb.setPolySigma(poly_sigma)
    fb.setFlags(flags)
    return fb.calc(prev, next, flow, stream)
