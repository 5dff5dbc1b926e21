"""numpy model of the reference's CUDA Dual TV-L1 path, ``cv::cuda::OpticalFlowDual_TVL1``
(modules/cudaoptflow/src/tvl1flow.cpp + src/cuda/tvl1flow.cu + cudawarping resize).

TEST INFRASTRUCTURE (see oracle/__init__.py).  This is the *semantics* the CUDA
kernels in opencv_contrib_b200/csrc implement (top-left aligned bilinear resize,
Keys a=-0.5 bicubic warp normalised by the weight sum with clamp addressing,
error sampled on the reference's cadence); kernels are compared with it at tight
tolerance, and with oracle/tvl1_cpu.py (the CPU reference path) at the stated
end-point-error tolerance.  It cannot be pinned against the CUDA reference
itself (that needs a GPU build of OpenCV, not available) -- "parity unpinned"
for this model; the CPU oracle is the parity anchor.

Citations: CO = opencv_contrib/modules/cudaoptflow, CW = opencv_contrib/modules/cudawarping.
"""
from __future__ import annotations

import numpy as np

F = np.float32
FLT_EPS = np.finfo(np.float32).eps


def cv_round(x: float) -> int:
    """cvRound / saturate_cast<int>(double): round half to even."""
    return int(np.rint(x))


class TVL1Params:
    """Defaults of cv::cuda::OpticalFlowDual_TVL1::create (CO/include/opencv2/cudaoptflow.hpp:375-385)."""

    def __init__(self, tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01,
                 iterations=300, scaleStep=0.8, gamma=0.0, useInitialFlow=False):
        self.tau, self.lambda_, self.theta = tau, lambda_, theta
        self.nscales, self.warps, self.epsilon = nscales, warps, epsilon
        self.iterations, self.scaleStep, self.gamma = iterations, scaleStep, gamma
        self.useInitialFlow = useInitialFlow


def level_sizes(h: int, w: int, nscales: int, scaleStep: float):
    """Pyramid sizes incl. the <16 px early stop (CO/src/tvl1flow.cpp:238-247; CW/src/resize.cpp:76-79)."""
    sizes = [(h, w)]
    for s in range(1, nscales):
        ph, pw = sizes[-1]
        nh, nw = cv_round(ph * scaleStep), cv_round(pw * scaleStep)
        sizes.append((nh, nw))
        if nw < 16 or nh < 16:
            return sizes[:s + 1], s  # level s is built but not used
    return sizes, nscales


def resize_linear(src: np.ndarray, dsize=None, fx: float = 0.0, fy: float = 0.0, dtype=F) -> np.ndarray:
    """cv::cuda::resize INTER_LINEAR, float C1 (CW/src/resize.cpp:57-106, CW/src/cuda/resize.cu:234-269).
    src = dst*scale (no half-pixel centre), scale = float(1/f), right/bottom taps clamped.  dtype: the arithmetic
    (np.float64 gives a double-precision yardstick; the scale stays the float value the kernel uses)."""
    H, W = src.shape
    if dsize is None:
        dw, dh = cv_round(W * fx), cv_round(H * fy)
    else:
        dh, dw = dsize
        fx, fy = dw / W, dh / H
    if (dh, dw) == (H, W):
        return src.copy()
    D = dtype
    sx, sy = D(F(1.0 / fx)), D(F(1.0 / fy))
    src_x = np.arange(dw, dtype=D) * sx
    src_y = np.arange(dh, dtype=D) * sy
    x1 = np.floor(src_x).astype(np.int64)
    y1 = np.floor(src_y).astype(np.int64)
    x2, y2 = x1 + 1, y1 + 1
    x2r, y2r = np.minimum(x2, W - 1), np.minimum(y2, H - 1)
    wx2 = (x2.astype(D) - src_x)[None, :]
    wx1 = (src_x - x1.astype(D))[None, :]
    wy2 = (y2.astype(D) - src_y)[:, None]
    wy1 = (src_y - y1.astype(D))[:, None]
    out = np.zeros((dh, dw), D)
    out = out + src[np.ix_(y1, x1)] * (wx2 * wy2)
    out = out + src[np.ix_(y1, x2r)] * (wx1 * wy2)
    out = out + src[np.ix_(y2r, x1)] * (wx2 * wy1)
    out = out + src[np.ix_(y2r, x2r)] * (wx1 * wy1)
    return out.astype(D)


def centered_gradient(src):
    """centeredGradientKernel (CO/src/cuda/tvl1flow.cu:59-69): clamped central difference * 0.5."""
    H, W = src.shape
    xs = np.arange(W)
    ys = np.arange(H)
    dx = F(0.5) * (src[:, np.minimum(xs + 1, W - 1)] - src[:, np.maximum(xs - 1, 0)])
    dy = F(0.5) * (src[np.minimum(ys + 1, H - 1), :] - src[np.maximum(ys - 1, 0), :])
    return dx.astype(F), dy.astype(F)


def bicubic_coeff(x):
    """bicubicCoeff (CO/src/cuda/tvl1flow.cu:89-104): Keys kernel, a = -0.5."""
    x = np.abs(x).astype(F)
    a = x * x * (F(1.5) * x - F(2.5)) + F(1.0)
    b = x * (x * (F(-0.5) * x + F(2.5)) - F(4.0)) + F(2.0)
    return np.where(x <= 1, a, np.where(x < 2, b, F(0))).astype(F)


def warp_backward(I0, I1, I1x, I1y, u1, u2):
    """warpBackwardKernel (CO/src/cuda/tvl1flow.cu:106-164).  Point/clamp texture reads; taps
    cx in [ceil(wx-2), floor(wx+2)] (<= 5), weights normalised by their sum."""
    H, W = I0.shape
    ys, xs = np.mgrid[0:H, 0:W]
    wx = xs.astype(F) + u1
    wy = ys.astype(F) + u2
    xmin = np.ceil(wx - F(2.0)).astype(np.int64)
    xmax = np.floor(wx + F(2.0)).astype(np.int64)
    ymin = np.ceil(wy - F(2.0)).astype(np.int64)
    ymax = np.floor(wy + F(2.0)).astype(np.int64)
    s = np.zeros((H, W), F)
    sx = np.zeros((H, W), F)
    sy = np.zeros((H, W), F)
    ws = np.zeros((H, W), F)
    for j in range(5):
        cy = ymin + j
        my = cy <= ymax
        cyc = np.clip(cy, 0, H - 1)
        ky = bicubic_coeff(wy - cy.astype(F))
        for i in range(5):
            cx = xmin + i
            m = my & (cx <= xmax)
            cxc = np.clip(cx, 0, W - 1)
            wgt = np.where(m, bicubic_coeff(wx - cx.astype(F)) * ky, F(0)).astype(F)
            s = s + wgt * I1[cyc, cxc]
            sx = sx + wgt * I1x[cyc, cxc]
            sy = sy + wgt * I1y[cyc, cxc]
            ws = ws + wgt
    coeff = F(1.0) / ws
    I1w = s * coeff
    I1wx = sx * coeff
    I1wy = sy * coeff
    grad = I1wx * I1wx + I1wy * I1wy
    rho = I1w - I1wx * u1 - I1wy * u2 - I0
    return I1w.astype(F), I1wx.astype(F), I1wy.astype(F), grad.astype(F), rho.astype(F)


def divergence(v1, v2):
    """divergence (CO/src/cuda/tvl1flow.cu:187-207)."""
    div = np.empty_like(v1)
    div[1:, 1:] = (v1[1:, 1:] - v1[1:, :-1]) + (v2[1:, 1:] - v2[:-1, 1:])
    div[1:, 0] = v1[1:, 0] + v2[1:, 0] - v2[:-1, 0]
    div[0, 1:] = v1[0, 1:] - v1[0, :-1] + v2[0, 1:]
    div[0, 0] = v1[0, 0] + v2[0, 0]
    return div


def estimate_u(I1wx, I1wy, grad, rho_c, p11, p12, p21, p22, p31, p32, u1, u2, u3, l_t, theta, gamma):
    """estimateUKernel (CO/src/cuda/tvl1flow.cu:209-288). Returns (u1, u2, u3, err_image)."""
    l_t, theta, gamma = F(l_t), F(theta), F(gamma)
    use_gamma = gamma != 0
    u3o = u3 if use_gamma else np.zeros_like(u1)
    rho = rho_c + (I1wx * u1 + I1wy * u2 + gamma * u3o)
    c1 = rho < -l_t * grad
    c2 = (~c1) & (rho > l_t * grad)
    c3 = (~c1) & (~c2) & (grad > FLT_EPS)
    with np.errstate(divide="ignore", invalid="ignore"):
        fi = np.where(c3, -rho / np.where(c3, grad, F(1)), F(0)).astype(F)
    sel = lambda a: np.where(c1, l_t * a, np.where(c2, -l_t * a, np.where(c3, fi * a, F(0)))).astype(F)
    v1 = u1 + sel(I1wx)
    v2 = u2 + sel(I1wy)
    n1 = v1 + theta * divergence(p11, p12)
    n2 = v2 + theta * divergence(p21, p22)
    n3 = None
    if use_gamma:
        v3 = u3o + sel(np.full_like(u1, gamma))
        n3 = (v3 + theta * divergence(p31, p32)).astype(F)
    err = (u1 - n1) * (u1 - n1) + (u2 - n2) * (u2 - n2)  # u3 not included on the GPU (:284-286)
    return n1.astype(F), n2.astype(F), n3, err.astype(F)


def estimate_dual(u1, u2, u3, p11, p12, p21, p22, p31, p32, taut, gamma):
    """estimateDualVariablesKernel (CO/src/cuda/tvl1flow.cu:313-348)."""
    taut = F(taut)

    def fwd(u):
        ux = np.zeros_like(u)
        uy = np.zeros_like(u)
        ux[:, :-1] = u[:, 1:] - u[:, :-1]
        uy[:-1, :] = u[1:, :] - u[:-1, :]
        return ux, uy

    def upd(pa, pb, u):
        ux, uy = fwd(u)
        g = np.hypot(ux, uy).astype(F)
        ng = F(1.0) + taut * g
        return ((pa + taut * ux) / ng).astype(F), ((pb + taut * uy) / ng).astype(F)

    p11, p12 = upd(p11, p12, u1)
    p21, p22 = upd(p21, p22, u2)
    if gamma != 0:
        p31, p32 = upd(p31, p32, u3)
    return p11, p12, p21, p22, p31, p32


def proc_one_scale(P: TVL1Params, I0, I1, u1, u2, u3, trace=None):
    """OpticalFlowDual_TVL1_Impl::procOneScale (CO/src/tvl1flow.cpp:304-382), incl. the error cadence."""
    h, w = I0.shape
    scaledEpsilon = P.epsilon * P.epsilon * (h * w)
    I1x, I1y = centered_gradient(I1)
    z = lambda: np.zeros((h, w), F)
    p11, p12, p21, p22 = z(), z(), z(), z()
    use_gamma = P.gamma != 0
    p31, p32 = (z(), z()) if use_gamma else (None, None)
    l_t = F(P.lambda_ * P.theta)
    taut = F(P.tau / P.theta)
    iters_run = []
    for _ in range(P.warps):
        _, I1wx, I1wy, grad, rho_c = warp_backward(I0, I1, I1x, I1y, u1, u2)
        error = np.finfo(np.float64).max
        prevError = 0.0
        n = 0
        while error > scaledEpsilon and n < P.iterations:
            calcError = (P.epsilon > 0) and bool(n & 1) and (prevError < scaledEpsilon)
            u1, u2, u3n, err = estimate_u(I1wx, I1wy, grad, rho_c, p11, p12, p21, p22, p31, p32,
                                          u1, u2, u3, l_t, P.theta, P.gamma)
            if use_gamma:
                u3 = u3n
            if calcError:
                error = float(err.astype(np.float64).sum())
                prevError = error
            else:
                error = np.finfo(np.float64).max
                prevError -= scaledEpsilon
            p11, p12, p21, p22, p31, p32 = estimate_dual(u1, u2, u3, p11, p12, p21, p22, p31, p32,
                                                         taut, P.gamma)
            n += 1
        iters_run.append(n)
    if trace is not None:
        trace.append(iters_run)
    return u1, u2, u3


def calc(I0: np.ndarray, I1: np.ndarray, P: TVL1Params | None = None, init_flow=None, trace=None):
    """OpticalFlowDual_TVL1_Impl::calc/calcImpl (CO/src/tvl1flow.cpp:170-302).
    Returns flow (H, W, 2) float32.  Note the reference's useInitialFlow quirk: flowx/flowy come
    from the buffer pool, so the caller's `flow` is never read (tvl1flow.cpp:175-179); the model
    (and the engine) instead read the caller's flow, which is what the API documents."""
    P = P or TVL1Params()
    assert I0.dtype in (np.uint8, np.float32) and I0.shape == I1.shape and I0.dtype == I1.dtype
    assert P.nscales > 0
    k = F(1.0) if I0.dtype == np.uint8 else F(255.0)
    h, w = I0.shape
    I0s, I1s = [I0.astype(F) * k], [I1.astype(F) * k]
    use_gamma = P.gamma != 0
    u1s = [np.zeros((h, w), F)]
    u2s = [np.zeros((h, w), F)]
    if P.useInitialFlow:
        u1s[0] = init_flow[..., 0].astype(F).copy()
        u2s[0] = init_flow[..., 1].astype(F).copy()
    nscales = P.nscales
    for s in range(1, nscales):
        a = resize_linear(I0s[s - 1], fx=P.scaleStep, fy=P.scaleStep)
        b = resize_linear(I1s[s - 1], fx=P.scaleStep, fy=P.scaleStep)
        I0s.append(a)
        I1s.append(b)
        if a.shape[1] < 16 or a.shape[0] < 16:
            nscales = s
            break
        if P.useInitialFlow:
            u1s.append(resize_linear(u1s[s - 1], fx=P.scaleStep, fy=P.scaleStep) * F(P.scaleStep))
            u2s.append(resize_linear(u2s[s - 1], fx=P.scaleStep, fy=P.scaleStep) * F(P.scaleStep))
        else:
            u1s.append(np.zeros(a.shape, F))
            u2s.append(np.zeros(a.shape, F))
    u3 = np.zeros(I0s[nscales - 1].shape, F) if use_gamma else None
    for s in range(nscales - 1, -1, -1):
        u1s[s], u2s[s], u3 = proc_one_scale(P, I0s[s], I1s[s], u1s[s], u2s[s], u3, trace)
        if s == 0:
            break
        dsz = I0s[s - 1].shape
        inv = F(1.0 / P.scaleStep)
        u1s[s - 1] = resize_linear(u1s[s], dsize=dsz) * inv
        u2s[s - 1] = resize_linear(u2s[s], dsize=dsz) * inv
        if use_gamma:
            u3 = resize_linear(u3, dsize=dsz)  # resized, not rescaled (tvl1flow.cpp:293-300)
    return np.stack([u1s[0], u2s[0]], axis=-1)
