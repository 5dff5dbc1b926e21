"""numpy model of the reference's CUDA Farneback path, ``cv::cuda::FarnebackOpticalFlow``
(modules/cudaoptflow/src/farneback.cpp + src/cuda/farneback.cu + cudawarping resize/pyrDown).

TEST INFRASTRUCTURE (see oracle/__init__.py).  The parity anchor for Farneback is the LIVE CPU
reference ``cv2.calcOpticalFlowFarneback`` (pinned in tests/test_oracle_cpu.py); this model restates
the CUDA reference's stage semantics (top-left resize, 5-plane stacked R/M, border weights,
replicate-border box filter) so individual kernels can be checked stage by stage.  It cannot be
pinned against the CUDA reference itself (no GPU OpenCV build) -- the end-to-end check against
cv2 is what carries the parity claim.

Citations: CO = opencv_contrib/modules/cudaoptflow.
"""
from __future__ import annotations

import numpy as np
import cv2

from .tvl1_gpu_model import resize_linear, cv_round

F = np.float32
OPTFLOW_USE_INITIAL_FLOW = 4
OPTFLOW_FARNEBACK_GAUSSIAN = 256
MIN_SIZE = 32          # CO/src/farneback.cpp:54
BORDER = np.array([0.14, 0.14, 0.4472, 0.4472, 0.4472, 1.0], F)  # CO/src/cuda/farneback.cu:246


class FarnebackParams:
    """Defaults of cv::cuda::FarnebackOpticalFlow::create (CO/include/opencv2/cudaoptflow.hpp:285-293)."""

    def __init__(self, numLevels=5, pyrScale=0.5, fastPyramids=False, winSize=13, numIters=10, polyN=5,
                 polySigma=1.1, flags=0):
        self.numLevels, self.pyrScale, self.fastPyramids = numLevels, pyrScale, fastPyramids
        self.winSize, self.numIters, self.polyN, self.polySigma, self.flags = winSize, numIters, polyN, polySigma, flags


def prepare_gaussian(n: int, sigma: float):
    """FarnebackOpticalFlowImpl::prepareGaussian (CO/src/farneback.cpp:209-260) + sigma rule (:269-270).
    Returns g, xg, xxg (index 0..n, float32) and ig11, ig03, ig33, ig55 (float32)."""
    if sigma < np.finfo(np.float32).eps:
        sigma = n * 0.3
    xs = np.arange(-n, n + 1)
    g = np.exp(-xs * xs / (2 * sigma * sigma)).astype(F)   # (float)std::exp(double)
    s = 0.0
    for v in g:
        s += float(v)
    s = 1.0 / s
    g = (g.astype(np.float64) * s).astype(F)
    xg = (xs.astype(F) * g).astype(F)                       # (float)(x*g[x]): int*float is a float multiply
    xxg = ((xs * xs).astype(F) * g).astype(F)
    G = np.zeros((6, 6), np.float64)
    for yi, y in enumerate(xs):
        for xi, x in enumerate(xs):
            gg = F(g[yi] * g[xi])  # g[y]*g[x]*x*x... is evaluated left to right in float, then added to double
            xf, yf = F(x), F(y)
            G[0, 0] += float(gg)
            G[1, 1] += float(F(F(gg * xf) * xf))
            G[3, 3] += float(F(F(F(F(gg * xf) * xf) * xf) * xf))
            G[5, 5] += float(F(F(F(F(gg * xf) * xf) * yf) * yf))
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    invG = np.linalg.inv(G)
    c = n
    return (g[c:], xg[c:], xxg[c:], F(invG[1, 1]), F(invG[0, 3]), F(invG[3, 3]), F(invG[5, 5]))


def poly_exp(src: np.ndarray, n: int, sigma: float) -> np.ndarray:
    """polynomialExpansion<polyN> (CO/src/cuda/farneback.cu:66-119).  Returns R (5, H, W) in src's dtype."""
    g, xg, xxg, ig11, ig03, ig33, ig55 = prepare_gaussian(n, sigma)
    H, W = src.shape
    ys = np.arange(H)
    r0 = src * g[0]
    r1 = np.zeros_like(src)
    r2 = np.zeros_like(src)
    for k in range(1, n + 1):
        t0 = src[np.maximum(ys - k, 0), :]
        t1 = src[np.minimum(ys + k, H - 1), :]
        r0 = r0 + g[k] * (t0 + t1)
        r1 = r1 + xg[k] * (t1 - t0)
        r2 = r2 + xxg[k] * (t0 + t1)
    xs = np.arange(W)

    def col(a, d):
        return a[:, np.clip(xs + d, 0, W - 1)]

    b1 = g[0] * r0
    b3 = g[0] * r1
    b5 = g[0] * r2
    b2 = np.zeros_like(src)
    b4 = np.zeros_like(src)
    b6 = np.zeros_like(src)
    for k in range(1, n + 1):
        b1 = b1 + (col(r0, k) + col(r0, -k)) * g[k]
        b4 = b4 + (col(r0, k) + col(r0, -k)) * xxg[k]
        b2 = b2 + (col(r0, k) - col(r0, -k)) * xg[k]
        b3 = b3 + (col(r1, k) + col(r1, -k)) * g[k]
        b6 = b6 + (col(r1, k) - col(r1, -k)) * xg[k]
        b5 = b5 + (col(r2, k) + col(r2, -k)) * g[k]
    R = np.stack([b3 * ig11, b2 * ig11, b1 * ig03 + b5 * ig33, b1 * ig03 + b4 * ig33, b6 * ig55]).astype(src.dtype)
    return R


def update_matrices(fx_, fy_, R0, R1) -> np.ndarray:
    """updateMatrices (CO/src/cuda/farneback.cu:156-241).  Returns M (5, H, W) in the flow's dtype."""
    D = fx_.dtype.type
    H, W = fx_.shape
    ys, xs = np.mgrid[0:H, 0:W]
    dx, dy = fx_, fy_
    fx = xs.astype(D) + dx
    fy = ys.astype(D) + dy
    x1 = np.floor(fx).astype(np.int64)
    y1 = np.floor(fy).astype(np.int64)
    fx = (fx - x1.astype(D)).astype(D)
    fy = (fy - y1.astype(D)).astype(D)
    inb = (x1 >= 0) & (y1 >= 0) & (x1 < W - 1) & (y1 < H - 1)
    x1c = np.clip(x1, 0, W - 2)
    y1c = np.clip(y1, 0, H - 2)
    a00 = (D(1) - fx) * (D(1) - fy)
    a01 = fx * (D(1) - fy)
    a10 = (D(1) - fx) * fy
    a11 = fx * fy

    def gather(P):
        return (a00 * P[y1c, x1c] + a01 * P[y1c, x1c + 1] + a10 * P[y1c + 1, x1c] + a11 * P[y1c + 1, x1c + 1]).astype(D)

    r2 = np.where(inb, gather(R1[0]), D(0)).astype(D)
    r3 = np.where(inb, gather(R1[1]), D(0)).astype(D)
    r4 = np.where(inb, (R0[2] + gather(R1[2])) * D(0.5), R0[2]).astype(D)
    r5 = np.where(inb, (R0[3] + gather(R1[3])) * D(0.5), R0[3]).astype(D)
    r6 = np.where(inb, (R0[4] + gather(R1[4])) * D(0.25), R0[4] * D(0.5)).astype(D)
    r2 = (R0[0] - r2) * D(0.5)
    r3 = (R0[1] - r3) * D(0.5)
    r2 = r2 + r4 * dy + r6 * dx
    r3 = r3 + r6 * dy + r5 * dx
    bs = 5
    B = BORDER.astype(D)
    scale = (B[np.minimum(xs, bs)] * B[np.minimum(ys, bs)] *
             B[np.minimum(W - xs - 1, bs)] * B[np.minimum(H - ys - 1, bs)]).astype(D)
    r2, r3, r4, r5, r6 = r2 * scale, r3 * scale, r4 * scale, r5 * scale, r6 * scale
    return np.stack([r4 * r4 + r6 * r6, (r4 + r5) * r6, r5 * r5 + r6 * r6, r4 * r2 + r6 * r3,
                     r6 * r2 + r5 * r3]).astype(D)


def update_flow(M):
    """updateFlow (CO/src/cuda/farneback.cu:267-286)."""
    D = M.dtype.type
    g11, g12, g22, h1, h2 = M
    det_inv = D(1.0) / (g11 * g22 - g12 * g12 + D(F(1e-3)))
    return ((g11 * h2 - g12 * h1) * det_inv).astype(D), ((g22 * h1 - g12 * h2) * det_inv).astype(D)


def _sep_filter(P, taps, border):
    """Shared shape of boxFilter5 / gaussianBlur(5): vertical pass into rows, then horizontal,
    symmetric pair order (CO/src/cuda/farneback.cu:357-412,455-492,539-595)."""
    H, W = P.shape[-2:]
    k = len(taps) - 1
    ys, xs = np.arange(H), np.arange(W)
    if border == "replicate":
        ry = lambda i: np.clip(i, 0, H - 1)
        rx = lambda i: np.clip(i, 0, W - 1)
    else:  # reflect101
        def refl(i, n):
            i = np.abs(i)
            return np.where(i >= n, 2 * n - 2 - i, i)
        ry = lambda i: refl(i, H)
        rx = lambda i: refl(i, W)
    row = P[..., :, :] * taps[0]
    for j in range(1, k + 1):
        row = row + (P[..., ry(ys - j), :] + P[..., ry(ys + j), :]) * taps[j]
    res = row * taps[0]
    for i in range(1, k + 1):
        res = res + (row[..., :, rx(xs - i)] + row[..., :, rx(xs + i)]) * taps[i]
    return res.astype(P.dtype)


def box_filter5(M, ksize_half):
    """boxFilter5 (CO/src/cuda/farneback.cu:357-412): plain sums then * 1/area, replicate border."""
    H, W = M.shape[-2:]
    ys, xs = np.arange(H), np.arange(W)
    row = M.copy()
    for j in range(1, ksize_half + 1):
        row = row + (M[:, np.clip(ys - j, 0, H - 1), :] + M[:, np.clip(ys + j, 0, H - 1), :])
    res = row.copy()
    for i in range(1, ksize_half + 1):
        res = res + (row[:, :, np.clip(xs - i, 0, W - 1)] + row[:, :, np.clip(xs + i, 0, W - 1)])
    inv = F(1.0 / ((1 + 2 * ksize_half) * (1 + 2 * ksize_half)))
    return (res * inv).astype(M.dtype)


def gaussian_kernel_half(ksize, sigma):
    g = cv2.getGaussianKernel(ksize, sigma, cv2.CV_32F).ravel()
    return g[ksize // 2:].astype(F)


def pyr_down(src):
    """cv::cuda::pyrDown f32 (cudawarping/src/cuda/pyr_down.cu:55-173): [1 4 6 4 1]/16 separable,
    BORDER_REFLECT101, dst = ((rows+1)/2, (cols+1)/2).  cv2.pyrDown uses the same kernel and
    default border (BORDER_REFLECT_101), so it doubles as the live check."""
    return cv2.pyrDown(src)


def level_sizes(H: int, W: int, P: FarnebackParams):
    """(rows, cols) of pyramid levels 0 (full size) .. top, as calc() builds them."""
    scale, cropped = 1.0, 0
    while cropped < P.numLevels:
        scale *= P.pyrScale
        if W * scale < MIN_SIZE or H * scale < MIN_SIZE:
            break
        cropped += 1
    sizes = [(H, W)]
    for k in range(1, cropped + 1):
        if P.fastPyramids:
            sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
        else:
            s = 1.0
            for _ in range(k):
                s *= P.pyrScale
            sizes.append((cv_round(H * s), cv_round(W * s)))
    return sizes


def calc(I0, I1, P: FarnebackParams | None = None, init_flow=None, stages=None, precision="f32"):
    """FarnebackOpticalFlowImpl::calc/calcImpl (CO/src/farneback.cpp:167-482).

    precision "f32" restates the kernels' float arithmetic; "f64" runs every operation in double (the constant tables
    -- polynomial-expansion and window kernels, border weights, resize scales -- keep the float values both use), a
    yardstick for how far float rounding alone moves the flow."""
    D = {"f32": F, "f64": np.float64}[precision]
    P = P or FarnebackParams()
    assert P.polyN in (5, 7)
    assert (not P.fastPyramids) or abs(P.pyrScale - 0.5) < 1e-6
    H, W = I0.shape
    frames = [I0.astype(D), I1.astype(D)]   # convertTo(CV_32F), no scaling (:342-345)
    scale = 1.0
    cropped = 0
    while cropped < P.numLevels:
        scale *= P.pyrScale
        if W * scale < MIN_SIZE or H * scale < MIN_SIZE:
            break
        cropped += 1
    pyr = None
    if P.fastPyramids:
        pyr = [[frames[0]], [frames[1]]]
        for i in range(1, cropped + 1):
            pyr[0].append(pyr_down(pyr[0][-1]))
            pyr[1].append(pyr_down(pyr[1][-1]))
    prev = None
    for k in range(cropped, -1, -1):
        scale = 1.0
        for _ in range(k):
            scale *= P.pyrScale
        sigma = (1.0 / scale - 1) * 0.5
        smooth = max(cv_round(sigma * 5) | 1, 3)
        w, h = cv_round(W * scale), cv_round(H * scale)
        if P.fastPyramids:
            h, w = pyr[0][k].shape
        if prev is None:
            if P.flags & OPTFLOW_USE_INITIAL_FLOW:
                fx = resize_linear(init_flow[..., 0].astype(D), dsize=(h, w), dtype=D) * F(scale)
                fy = resize_linear(init_flow[..., 1].astype(D), dsize=(h, w), dtype=D) * F(scale)
            else:
                fx = np.zeros((h, w), D)
                fy = np.zeros((h, w), D)
        else:
            fx = resize_linear(prev[0], dsize=(h, w), dtype=D) * F(1.0 / P.pyrScale)
            fy = resize_linear(prev[1], dsize=(h, w), dtype=D) * F(1.0 / P.pyrScale)
        R = []
        for i in range(2):
            if P.fastPyramids:
                lvl = pyr[i][k]
            else:
                g = gaussian_kernel_half(smooth, sigma)
                blurred = _sep_filter(frames[i], g, "reflect101")
                lvl = resize_linear(blurred, dsize=(h, w), dtype=D)
            R.append(poly_exp(lvl, P.polyN, P.polySigma))
            if stages is not None:
                stages.setdefault("level_image", {})[(k, i)] = lvl
                stages.setdefault("R", {})[(k, i)] = R[-1]
        M = update_matrices(fx, fy, R[0], R[1])
        if stages is not None:
            stages.setdefault("M0", {})[k] = M
        gk = None
        if P.flags & OPTFLOW_FARNEBACK_GAUSSIAN:
            gk = gaussian_kernel_half(P.winSize, float(F(P.winSize // 2 * F(0.3))))
        for it in range(P.numIters):
            if gk is not None:
                M = _sep_filter(M, gk, "replicate")
            else:
                M = box_filter5(M, P.winSize // 2)
            fx, fy = update_flow(M)
            if it < P.numIters - 1:
                M = update_matrices(fx, fy, R[0], R[1])
        prev = (fx, fy)
        if stages is not None:
            stages.setdefault("flow", {})[k] = np.stack([fx, fy], -1)
    return np.stack(prev, axis=-1)
