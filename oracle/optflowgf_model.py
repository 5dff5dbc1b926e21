"""The video module's Farneback flow (cv::calcOpticalFlowFarneback, cv::FarnebackOpticalFlow) restated in numpy with
cv2's own types, as cv2 4.x computes it on its portable path (``cv2.setUseOptimized(False)`` and
``cv2.ipp.setUseIPP(False)``: the SSE baseline code, the same on every x86-64 host and for every thread count).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Every rule below is pinned against the live cv2 by
tests/test_optflowgf_model_cpu.py; the engine (opencv_contrib_b200/csrc/optflowgf.cu, built with -fmad=false) rounds
where this model rounds.

* Levels: ``scale *= pyrScale`` while ``cols*scale`` and ``rows*scale`` stay >= 32, at most ``numLevels`` times.  Level
  k (scale = pyrScale^k) is built from the full-size frame converted to float: GaussianBlur with sigma
  (1/scale - 1)/2 and ksize max(cvRound(5 sigma) | 1, 3), reflect-101 border, then resize INTER_LINEAR to
  (cvRound(cols*scale), cvRound(rows*scale)).  Level 0 is blurred too, by getGaussianKernel(3, 0) = [1/4, 1/2, 1/4].
* GaussianBlur of a float plane: rows for ksize <= 5 ``kc x + k1 (l1 + r1) + k2 (l2 + r2)``, for larger kernels the
  sequential ``k0 x0 + k1 x1 + ...``; columns always ``kc x + sum k_i (up_i + down_i)``.
* resize INTER_LINEAR: centre-aligned, ``fx = float((d + 0.5) / (dst/src) - 0.5)``, horizontal ``s0 (1 - fx) + s1 fx``
  then vertical the same, all float.  Horizontally a tap outside the source moves to the edge with fraction 0;
  vertically the fraction stays and only the row indices clamp (upscales differ there).  An exact 2x downscale on
  both axes is OpenCV's fast INTER_AREA instead: for one channel ``((a + b) + (c + d)) * 0.25`` on the first
  4*floor(cols/4) columns and the generic ``(((a + b) + c) + d) * 0.25`` on the rest and on 2 channels.
* resize INTER_AREA (the initial flow to the coarsest level): integer factors sum the block row-major as
  ``sum += ((a + b) + c) + d`` per 4 taps, then times float(1/area); other factors use computeResizeAreaTab's float
  weights, a horizontal sum from 0 and a vertical sum from the first weighted row.
* Polynomial expansion, radius polyN: float vertical pass with clamped rows, double horizontal pass of float
  products with replicated columns; tables from FarnebackPrepareGaussian (float taps, double sums, Cholesky inverse).
* updateMatrices: float, bilinear gather of R1 at x + flow, border weights {0.14, 0.14, 0.4472, 0.4472, 0.4472}
  on the 5 pixels next to each edge (for sides below 10 pixels, only where both edges' bands overlap).
* Box window: double running sums; the vertical sum adds the float difference of two M rows, the horizontal sum
  the double difference of two column sums, both starting from ``first*(m+2) + next m-1``; 2x2 solve in double with
  ``+1e-3``.  m = winSize/2, scale 1/winSize^2 (an even winSize keeps the 2m+1 window).
* Gaussian window: float sums over ``exp(-i^2/(2 sigma^2))``, sigma = 0.3 m, vertical then horizontal, replicated
  borders; the solve in double on the float sums.
* cv2 updates M in row stripes during the next solve, on rows that have left its window; a full pass after each
  solve but the last is the same.
* Prolongation: resize INTER_LINEAR of the 2-channel flow, then ``float(x * float(1/pyrScale)) + 0.f``.
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
f64 = np.float64

OPTFLOW_USE_INITIAL_FLOW = 4
OPTFLOW_FARNEBACK_GAUSSIAN = 256
MIN_SIZE = 32
BORDER = (0.14, 0.14, 0.4472, 0.4472, 0.4472)


def cv_round(x: float) -> int:
    """cvRound: round half to even."""
    return int(round(x))


def reflect101(p, n):
    p = np.asarray(p, dtype=np.int64).copy()
    if n == 1:
        return np.zeros_like(p)
    while True:
        bad = (p < 0) | (p >= n)
        if not bad.any():
            return p
        neg = p < 0
        p[neg] = -p[neg]
        pos = p >= n
        p[pos] = 2 * (n - 1) - p[pos]


# --------------------------------------------------------------------------------------------------------- tables


def gaussian_kernel(n: int, sigma: float) -> np.ndarray:
    """getGaussianKernel(n, sigma, CV_32F): the fixed tables for sigma <= 0 and n <= 7, else exp in double,
    normalised, stored as float."""
    fixed = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
             7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125]}
    if sigma <= 0 and n in fixed:
        return np.array(fixed[n], f32)
    sx = sigma if sigma > 0 else n * 0.15 + 0.35
    s2 = -0.125 / (sx * sx)
    h = (n - 1) // 2
    vals = [math.exp(float(x * x) * s2) for x in range(1 - n, 1 - n + 2 * h, 2)]
    tot = sum(vals) * 2.0 + 1.0 + (1.0 if n % 2 == 0 else 0.0)
    mul = 1.0 / tot
    out = [v * mul for v in vals]
    mid = [mul] * (2 if n % 2 == 0 else 1)
    return np.array(out + mid + out[::-1], f32)


def level_blur(scale: float) -> tuple[float, int]:
    sigma = (1.0 / scale - 1.0) * 0.5
    return sigma, max(cv_round(sigma * 5) | 1, 3)


def _chol_inv(G: list[list[float]]) -> list[list[float]]:
    """cv::invert(DECOMP_CHOLESKY) of a 6x6 double matrix (hal Cholesky with the identity as right-hand side)."""
    m = len(G)
    L = [row[:] for row in G]
    b = [[1.0 if i == j else 0.0 for j in range(m)] for i in range(m)]
    for i in range(m):
        for j in range(i):
            s = L[i][j]
            for k in range(j):
                s -= L[i][k] * L[j][k]
            L[i][j] = s * L[j][j]
        s = L[i][i]
        for k in range(i):
            t = L[i][k]
            s -= t * t
        L[i][i] = 1.0 / math.sqrt(s)
    for i in range(m):
        for j in range(m):
            s = b[i][j]
            for k in range(i):
                s -= L[i][k] * b[k][j]
            b[i][j] = s * L[i][i]
    for i in range(m - 1, -1, -1):
        for j in range(m):
            s = b[i][j]
            for k in range(m - 1, i, -1):
                s -= L[k][i] * b[k][j]
            b[i][j] = s * L[i][i]
    return b


def poly_tables(n: int, sigma: float):
    """FarnebackPrepareGaussian: float g, xg, xxg over -n..n (index n + x) and the double ig11, ig03, ig33, ig55."""
    if sigma < float(np.finfo(f32).eps):
        sigma = n * 0.3
    g = [f32(math.exp(-x * x / (2 * sigma * sigma))) for x in range(-n, n + 1)]
    s = 0.0
    for v in g:
        s += float(v)
    s = 1.0 / s
    g = [f32(float(v) * s) for v in g]
    xg = [f32(x * float(g[x + n])) for x in range(-n, n + 1)]
    xxg = [f32(x * x * float(g[x + n])) for x in range(-n, n + 1)]
    G = [[0.0] * 6 for _ in range(6)]
    for y in range(-n, n + 1):
        for x in range(-n, n + 1):
            gyx = f32(g[y + n] * g[x + n])
            G[0][0] += float(gyx)
            G[1][1] += float(f32(f32(gyx * f32(x)) * f32(x)))
            G[3][3] += float(f32(f32(f32(f32(gyx * f32(x)) * f32(x)) * f32(x)) * f32(x)))
            G[5][5] += float(f32(f32(f32(f32(gyx * f32(x)) * f32(x)) * f32(y)) * f32(y)))
    G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1]
    G[4][4] = G[3][3]
    G[3][4] = G[4][3] = G[5][5]
    iG = _chol_inv(G)
    return (np.array(g, f32), np.array(xg, f32), np.array(xxg, f32),
            (iG[1][1], iG[0][3], iG[3][3], iG[5][5]))


def window_kernel(m: int) -> np.ndarray:
    """FarnebackUpdateFlow_GaussianBlur's taps 0..m: exp(-i^2/(2 sigma^2)) as float, normalised in double."""
    sigma = m * 0.3
    k = [f32(1.0)]
    s = 1.0
    for i in range(1, m + 1):
        t = f32(math.exp(-i * i / (2 * sigma * sigma)))
        k.append(t)
        s += float(f32(t * f32(2)))
    s = 1.0 / s
    return np.array([f32(float(v) * s) for v in k], f32)


# ------------------------------------------------------------------------------------------------ image primitives


def gaussian_blur(img: np.ndarray, ksize: int, sigma: float) -> np.ndarray:
    """GaussianBlur(float plane, (ksize, ksize), sigma, sigma), reflect-101 border, portable path."""
    a = np.asarray(img, f32)
    h, w = a.shape
    k = gaussian_kernel(ksize, sigma)
    r = ksize // 2
    xs = np.arange(w)
    if ksize <= 5:
        t = k[r] * a
        for i in range(1, r + 1):
            t = t + k[r + i] * (a[:, reflect101(xs - i, w)] + a[:, reflect101(xs + i, w)])
    else:
        t = k[0] * a[:, reflect101(xs - r, w)]
        for i in range(1, ksize):
            t = t + k[i] * a[:, reflect101(xs - r + i, w)]
    ys = np.arange(h)
    o = k[r] * t
    for i in range(1, r + 1):
        o = o + k[r + i] * (t[reflect101(ys - i, h)] + t[reflect101(ys + i, h)])
    return o.astype(f32)


def _linear_axis(n_src: int, n_dst: int, clamp: bool):
    """Source taps and fraction per destination index.  The horizontal axis (clamp) moves a tap outside the source
    onto the edge with fraction 0; the vertical one keeps the fraction and clamps the two row indices."""
    scale = 1.0 / (n_dst / n_src)
    i0, i1, fr = [], [], []
    for d in range(n_dst):
        f = f32((d + 0.5) * scale - 0.5)
        s = math.floor(f)
        f = f32(f - f32(s))
        if clamp and s < 0:
            s, f = 0, f32(0)
        if clamp and s >= n_src - 1:
            s, f = n_src - 1, f32(0)
        i0.append(min(max(s, 0), n_src - 1))
        i1.append(min(max(s + 1, 0), n_src - 1))
        fr.append(f)
    return np.array(i0), np.array(i1), np.array(fr, f32)


def _area_fast(src: np.ndarray, rows: int, cols: int) -> np.ndarray:
    """OpenCV's fast INTER_AREA for integer factors: block taps summed row-major, four per step, times 1/area."""
    h, w = src.shape[:2]
    sy, sx = h // rows, w // cols
    taps = [src[dy: dy + sy * rows: sy, dx: dx + sx * cols: sx] for dy in range(sy) for dx in range(sx)]
    acc = np.zeros_like(taps[0])
    k = 0
    while k + 4 <= len(taps):
        acc = acc + (((taps[k] + taps[k + 1]) + taps[k + 2]) + taps[k + 3])
        k += 4
    for t in taps[k:]:
        acc = acc + t
    out = (acc * f32(1.0 / (sx * sy))).astype(f32)
    if sx == 2 and sy == 2 and src.ndim == 2:
        # the 1-channel 2x2 vector path, 4 columns at a time: ((a + b) + (c + d)) * 0.25
        v = cols - cols % 4
        s = src[: 2 * rows, : 2 * v]
        out[:, :v] = ((s[0::2, 0::2] + s[0::2, 1::2]) + (s[1::2, 0::2] + s[1::2, 1::2])) * f32(0.25)
    return out


def _exact_integer(n_src: int, n_dst: int):
    s = 1.0 / (n_dst / n_src)
    i = int(s)
    return i if abs(s - i) < np.finfo(f64).eps else 0


def resize_linear(src: np.ndarray, rows: int, cols: int) -> np.ndarray:
    """cv::resize(INTER_LINEAR) of a float plane or 2-channel field."""
    a = np.asarray(src, f32)
    h, w = a.shape[:2]
    if (h, w) == (rows, cols):
        return a.copy()
    if _exact_integer(w, cols) == 2 and _exact_integer(h, rows) == 2:
        return _area_fast(a, rows, cols)
    x0, x1, fx = _linear_axis(w, cols, True)
    y0, y1, fy = _linear_axis(h, rows, False)
    ex = (slice(None), None) if a.ndim == 3 else (slice(None),)
    one = f32(1)
    t = a[:, x0] * (one - fx)[ex] + a[:, x1] * fx[ex]
    ey = (slice(None), None, None) if a.ndim == 3 else (slice(None), None)
    return (t[y0] * (one - fy)[ey] + t[y1] * fy[ey]).astype(f32)


def _area_tab(n_src: int, n_dst: int):
    scale = 1.0 / (n_dst / n_src)
    tab = []
    for d in range(n_dst):
        f1 = d * scale
        f2 = f1 + scale
        cw = min(scale, n_src - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, n_src - 1)
        s1 = min(s1, s2)
        t = []
        if s1 - f1 > 1e-3:
            t.append((s1 - 1, f32((s1 - f1) / cw)))
        for s in range(s1, s2):
            t.append((s, f32(1.0 / cw)))
        if f2 - s2 > 1e-3:
            t.append((s2, f32(min(min(f2 - s2, 1.0), cw) / cw)))
        tab.append(t)
    return tab


def resize_area(src: np.ndarray, rows: int, cols: int) -> np.ndarray:
    """cv::resize(INTER_AREA) of a float plane or 2-channel field to a size no larger."""
    a = np.asarray(src, f32)
    h, w = a.shape[:2]
    if (h, w) == (rows, cols):
        return a.copy()
    if _exact_integer(w, cols) and _exact_integer(h, rows):
        return _area_fast(a, rows, cols)
    xt, yt = _area_tab(w, cols), _area_tab(h, rows)
    buf = np.zeros((h, cols) + a.shape[2:], f32)
    for dx, t in enumerate(xt):
        acc = np.zeros((h,) + a.shape[2:], f32)
        for sx, al in t:
            acc = acc + a[:, sx] * al
        buf[:, dx] = acc
    out = np.zeros((rows, cols) + a.shape[2:], f32)
    for dy, t in enumerate(yt):
        acc = None
        for sy, b in t:
            acc = b * buf[sy] if acc is None else acc + b * buf[sy]
        out[dy] = acc
    return out


# ------------------------------------------------------------------------------------------------------ Farneback


def poly_exp(img: np.ndarray, n: int, sigma: float) -> np.ndarray:
    """FarnebackPolyExp: (h, w, 5) float32 coefficients [r3, r2, r5, r4, r6] as cv2 stores them."""
    src = np.asarray(img, f32)
    h, w = src.shape
    g, xg, xxg, (ig11, ig03, ig33, ig55) = poly_tables(n, sigma)
    ys = np.arange(h)
    r0 = src * g[n]
    r1 = np.zeros_like(src)
    r2 = np.zeros_like(src)
    for k in range(1, n + 1):
        s0 = src[np.maximum(ys - k, 0)]
        s1 = src[np.minimum(ys + k, h - 1)]
        p = s0 + s1
        r0 = r0 + g[n + k] * p
        r1 = r1 + xg[n + k] * (s1 - s0)
        r2 = r2 + xxg[n + k] * p
    xs = np.arange(w)
    b1 = (r0 * g[n]).astype(f64)
    b3 = (r1 * g[n]).astype(f64)
    b5 = (r2 * g[n]).astype(f64)
    b2 = np.zeros((h, w), f64)
    b4 = np.zeros((h, w), f64)
    b6 = np.zeros((h, w), f64)
    for k in range(1, n + 1):
        R, L = np.minimum(xs + k, w - 1), np.maximum(xs - k, 0)
        tg = (r0[:, R] + r0[:, L]).astype(f64)
        g0 = g[n + k]
        b1 = b1 + tg * f64(g0)
        b4 = b4 + tg * f64(xxg[n + k])
        b2 = b2 + ((r0[:, R] - r0[:, L]) * xg[n + k]).astype(f64)
        b3 = b3 + ((r1[:, R] + r1[:, L]) * g0).astype(f64)
        b6 = b6 + ((r1[:, R] - r1[:, L]) * xg[n + k]).astype(f64)
        b5 = b5 + ((r2[:, R] + r2[:, L]) * g0).astype(f64)
    out = np.empty((h, w, 5), f32)
    out[..., 1] = b2 * ig11
    out[..., 0] = b3 * ig11
    out[..., 3] = b1 * ig03 + b4 * ig33
    out[..., 2] = b1 * ig03 + b5 * ig33
    out[..., 4] = b6 * ig55
    return out


def update_matrices(R0: np.ndarray, R1: np.ndarray, flow: np.ndarray) -> np.ndarray:
    """FarnebackUpdateMatrices over the whole field: (h, w, 5) float32 [G11, G12, G22, h1, h2]."""
    h, w = flow.shape[:2]
    dx, dy = flow[..., 0], flow[..., 1]
    ys, xs = np.mgrid[0:h, 0:w]
    with np.errstate(invalid="ignore", over="ignore"):
        fx = xs.astype(f32) + dx
        fy = ys.astype(f32) + dy
        x1f, y1f = np.floor(fx), np.floor(fy)
        inside = (x1f >= 0) & (x1f < w - 1) & (y1f >= 0) & (y1f < h - 1)
        x1 = np.where(inside, x1f, 0).astype(np.int64)
        y1 = np.where(inside, y1f, 0).astype(np.int64)
        fx = (fx - x1f).astype(f32)
        fy = (fy - y1f).astype(f32)
    one = f32(1)
    a00, a01 = (one - fx) * (one - fy), fx * (one - fy)
    a10, a11 = (one - fx) * fy, fx * fy
    x2, y2 = np.minimum(x1 + 1, w - 1), np.minimum(y1 + 1, h - 1)
    P00, P01, P10, P11 = R1[y1, x1], R1[y1, x2], R1[y2, x1], R1[y2, x2]
    r = [((a00 * P00[..., c] + a01 * P01[..., c]) + a10 * P10[..., c]) + a11 * P11[..., c] for c in range(5)]
    half, quarter = f32(0.5), f32(0.25)
    r2 = np.where(inside, r[0], f32(0))
    r3 = np.where(inside, r[1], f32(0))
    r4 = np.where(inside, (R0[..., 2] + r[2]) * half, R0[..., 2])
    r5 = np.where(inside, (R0[..., 3] + r[3]) * half, R0[..., 3])
    r6 = np.where(inside, (R0[..., 4] + r[4]) * quarter, R0[..., 4] * half)
    r2 = (R0[..., 0] - r2) * half
    r3 = (R0[..., 1] - r3) * half
    r2 = r2 + (r4 * dy + r6 * dx)
    r3 = r3 + (r6 * dy + r5 * dx)
    b = np.array(BORDER, f32)
    sx_lo = np.ones(w, f32)
    sx_hi = np.ones(w, f32)
    sy_lo = np.ones(h, f32)
    sy_hi = np.ones(h, f32)
    for i in range(min(5, w)):
        sx_lo[i] = b[i]
        sx_hi[w - 1 - i] = b[i]
    for i in range(min(5, h)):
        sy_lo[i] = b[i]
        sy_hi[h - 1 - i] = b[i]
    scale = ((sx_lo[None, :] * sx_hi[None, :]) * sy_lo[:, None]) * sy_hi[:, None]
    # cv2's test (unsigned)(x - 5) >= (unsigned)(width - 10), which for a width below 10 selects only
    # width - 5 <= x < 5
    ex = ((xs[0] - 5) & 0xFFFFFFFF) >= ((w - 10) & 0xFFFFFFFF)
    ey = ((ys[:, 0] - 5) & 0xFFFFFFFF) >= ((h - 10) & 0xFFFFFFFF)
    edge = ex[None, :] | ey[:, None]
    r2, r3, r4, r5, r6 = (np.where(edge, v * scale, v) for v in (r2, r3, r4, r5, r6))
    M = np.empty((h, w, 5), f32)
    M[..., 0] = r4 * r4 + r6 * r6
    M[..., 1] = (r4 + r5) * r6
    M[..., 2] = r5 * r5 + r6 * r6
    M[..., 3] = r4 * r2 + r6 * r3
    M[..., 4] = r6 * r2 + r5 * r3
    return M


def _solve(g11, g12, g22, h1, h2):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        idet = 1.0 / (g11 * g22 - g12 * g12 + 1e-3)
        return np.stack([((g11 * h2 - g12 * h1) * idet).astype(f32), ((g22 * h1 - g12 * h2) * idet).astype(f32)], -1)


def solve_box(M: np.ndarray, win: int) -> np.ndarray:
    """FarnebackUpdateFlow_Blur's flow: sequential double running sums are cumulative sums of per-step differences."""
    h, w = M.shape[:2]
    m = win // 2
    scale = 1.0 / (win * win)
    Mf = M.reshape(h, w * 5)
    ys = np.arange(h)
    head = [(Mf[0] * f32(m + 2)).astype(f64)] + [Mf[min(y, h - 1)].astype(f64) for y in range(1, m)]
    diff = (Mf[np.minimum(ys + m, h - 1)] - Mf[np.maximum(ys - m - 1, 0)]).astype(f64)
    vs = np.cumsum(np.concatenate([np.stack(head), diff]), axis=0)[len(head):].reshape(h, w, 5)
    xs = np.arange(w)
    hh = [vs[:, 0] * f64(m + 2)] + [vs[:, min(x, w - 1)] for x in range(1, m)]
    hd = vs[:, np.minimum(xs + m, w - 1)] - vs[:, np.maximum(xs - m - 1, 0)]
    hs = np.cumsum(np.concatenate([np.stack(hh, 1), hd], 1), axis=1)[:, len(hh):] * scale
    return _solve(*(hs[..., c] for c in range(5)))


def solve_gauss(M: np.ndarray, win: int) -> np.ndarray:
    """FarnebackUpdateFlow_GaussianBlur's flow."""
    h, w = M.shape[:2]
    m = win // 2
    k = window_kernel(m)
    ys, xs = np.arange(h), np.arange(w)
    v = M * k[0]
    for i in range(1, m + 1):
        v = v + (M[np.minimum(ys + i, h - 1)] + M[np.maximum(ys - i, 0)]) * k[i]
    s = v * k[0]
    for i in range(1, m + 1):
        s = s + k[i] * (v[:, np.maximum(xs - i, 0)] + v[:, np.minimum(xs + i, w - 1)])
    s = s.astype(f64)
    return _solve(*(s[..., c] for c in range(5)))


def scale_flow(flow: np.ndarray, s: float) -> np.ndarray:
    """Mat *= s on a float field: convertTo(alpha = s) rounds float(x * float(s)) + 0.f; *= 1 in place is a no-op."""
    if s == 1.0:
        return flow.copy()
    return (flow * f32(s)) + f32(0)


def level_count(rows: int, cols: int, pyr_scale: float, levels: int) -> int:
    scale, k = 1.0, 0
    while k < levels:
        scale *= pyr_scale
        if cols * scale < MIN_SIZE or rows * scale < MIN_SIZE:
            break
        k += 1
    return k


def calc(prev, nxt, flow=None, pyr_scale=0.5, levels=5, winsize=13, iterations=10, poly_n=5, poly_sigma=1.1,
         flags=0, trace=None):
    """cv2.calcOpticalFlowFarneback(prev, next, flow, ...) on the portable path; returns (h, w, 2) float32."""
    I = [np.asarray(prev).astype(f32), np.asarray(nxt).astype(f32)]
    rows, cols = I[0].shape
    L = level_count(rows, cols, pyr_scale, levels)
    prev_flow = None
    out = None
    for k in range(L, -1, -1):
        scale = 1.0
        for _ in range(k):
            scale *= pyr_scale
        sigma, ks = level_blur(scale)
        width, height = cv_round(cols * scale), cv_round(rows * scale)
        if prev_flow is None:
            if flags & OPTFLOW_USE_INITIAL_FLOW:
                fl = scale_flow(resize_area(np.asarray(flow, f32), height, width), scale)
            else:
                fl = np.zeros((height, width, 2), f32)
        else:
            fl = scale_flow(resize_linear(prev_flow, height, width), 1.0 / pyr_scale)
        R = [poly_exp(resize_linear(gaussian_blur(im, ks, sigma), height, width), poly_n, poly_sigma) for im in I]
        M = update_matrices(R[0], R[1], fl)
        for i in range(iterations):
            fl = (solve_gauss if flags & OPTFLOW_FARNEBACK_GAUSSIAN else solve_box)(M, winsize)
            if i < iterations - 1:
                M = update_matrices(R[0], R[1], fl)
        if trace is not None:
            trace.append(dict(level=k, scale=scale, size=(height, width), ksize=ks, sigma=sigma))
        prev_flow = fl
        out = fl
    return out
