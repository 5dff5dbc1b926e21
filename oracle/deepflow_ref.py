"""The optflow module's DeepFlow driver (``cv::optflow::createOptFlow_DeepFlow``, modules/optflow/src/deepflow.cpp:116-169)
restated over the live cv2 wheel.

TEST INFRASTRUCTURE (see oracle/__init__.py).  deepflow.cpp is only a driver: Gaussian pre-smoothing, a pyramid with a
0.95 step built by ``cv::resize``, and one ``cv::VariationalRefinement`` call per level, coarse to fine.  Every one of
those is in the installed cv2, so this is the reference's own arithmetic for everything but the driver's few lines,
which are restated here one for one:

* inputs converted to float32 without scaling;
* ``GaussianBlur`` with ``kernelLen = floor(3 * sigma) * 2 + 1`` (3 at sigma 0.6), default border; ``sigma`` is a float
  member (0.6f), widened to double by the call;
* ``nextSize = (int)(prev * 0.95f + 0.5f)`` in float; stop when a side is ``<= minSize``; at most ``maxLayers`` levels
  below the source (buildPyramid pushes the source, then loops ``maxLayers`` times), so ``maxLayers + 1`` in all;
  each level is ``resize(INTER_LINEAR)`` of the previous one;
* zero flow at the coarsest level; per level ``VariationalRefinement`` with alpha ``4 * alpha``, delta ``delta / 3``,
  gamma ``gamma / 3`` (all float), ``fixedPointIterations``, ``sorIterations`` and ``omega``;
* prolongation: ``resize`` of the CV_32FC2 flow, then ``*= 1.0f / 0.95f``.

``solver`` replaces the per-level ``VariationalRefinement`` call (the tests pass the numpy model's solver there).
"""
from __future__ import annotations

import dataclasses
import math

import cv2
import numpy as np

F = np.float32


@dataclasses.dataclass(frozen=True)
class DeepFlowParams:
    """Fields and defaults of the ``OpticalFlowDeepFlow`` constructor (deepflow.cpp:62-73)."""
    sigma: float = 0.6
    min_size: int = 25
    downscale_factor: float = 0.95
    fixed_point_iterations: int = 5
    sor_iterations: int = 25
    alpha: float = 1.0
    delta: float = 0.5
    gamma: float = 5.0
    omega: float = 1.6
    max_layers: int = 200


def float_sigma(sigma: float) -> float:
    """The reference's float member, as the double GaussianBlur / getGaussianKernel receive it."""
    return float(F(sigma))


def kernel_len(sigma: float) -> int:
    return int(math.floor(F(3) * F(sigma))) * 2 + 1


def pyramid_sizes(rows: int, cols: int, p: DeepFlowParams = DeepFlowParams()) -> list[tuple[int, int]]:
    """(rows, cols) of every level, finest first (deepflow.cpp buildPyramid)."""
    sizes = [(rows, cols)]
    f = F(p.downscale_factor)
    for _ in range(p.max_layers):
        pr, pc = sizes[-1]
        nc = int(F(F(pc) * f) + F(0.5))
        nr = int(F(F(pr) * f) + F(0.5))
        if nr <= p.min_size or nc <= p.min_size:
            break
        sizes.append((nr, nc))
    return sizes


def solver_params(p: DeepFlowParams) -> dict:
    """The float parameters deepflow.cpp hands to VariationalRefinement."""
    return dict(alpha=float(F(4.0 * F(p.alpha))), delta=float(F(F(p.delta) / F(3.0))),
                gamma=float(F(F(p.gamma) / F(3.0))), omega=float(F(p.omega)),
                fixed_point_iterations=p.fixed_point_iterations, sor_iterations=p.sor_iterations)


def cv2_solver(I0: np.ndarray, I1: np.ndarray, flow: np.ndarray, sp: dict) -> np.ndarray:
    """One ``cv::VariationalRefinement::calc`` call; flow (h, w, 2) float32 in, refined flow out."""
    vr = cv2.VariationalRefinement_create()
    vr.setAlpha(sp["alpha"])
    vr.setDelta(sp["delta"])
    vr.setGamma(sp["gamma"])
    vr.setOmega(sp["omega"])
    vr.setFixedPointIterations(sp["fixed_point_iterations"])
    vr.setSorIterations(sp["sor_iterations"])
    return vr.calc(I0, I1, np.array(flow, dtype=np.float32, order="C"))  # calc refines its argument in place


def calc(I0: np.ndarray, I1: np.ndarray, p: DeepFlowParams = DeepFlowParams(), solver=cv2_solver) -> np.ndarray:
    """DeepFlow of the pair; (h, w, 2) float32."""
    a = I0.astype(np.float32)
    b = I1.astype(np.float32)
    k = kernel_len(p.sigma)
    sg = float_sigma(p.sigma)
    a = cv2.GaussianBlur(a, (k, k), sg, sigmaY=sg)
    b = cv2.GaussianBlur(b, (k, k), sg, sigmaY=sg)
    sizes = pyramid_sizes(*a.shape, p)
    pyr0, pyr1 = [a], [b]
    for r, c in sizes[1:]:
        pyr0.append(cv2.resize(pyr0[-1], (c, r), interpolation=cv2.INTER_LINEAR))
        pyr1.append(cv2.resize(pyr1[-1], (c, r), interpolation=cv2.INTER_LINEAR))
    sp = solver_params(p)
    r, c = sizes[-1]
    flow = np.zeros((r, c, 2), np.float32)
    mul = F(F(1.0) / F(p.downscale_factor))
    for i in range(len(sizes) - 1, -1, -1):
        if i < len(sizes) - 1:
            r, c = sizes[i]
            flow = cv2.resize(flow, (c, r), interpolation=cv2.INTER_LINEAR)
            flow = (flow * mul).astype(np.float32)
        flow = solver(pyr0[i], pyr1[i], flow, sp)
    return flow
