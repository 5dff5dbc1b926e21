"""Float32 restatement of cudaimgproc's corner classes, one operation at a time, in the order the engine
(opencv_contrib_b200/csrc/corners.cu, built with -fmad=false) evaluates them.

Rounding policy: every +, * and sqrt rounds once to float32 (numpy float32 arithmetic); there is no FMA contraction on
either side, so the engine equals this model bit for bit.

- response(): CornerBase (modules/cudaimgproc/src/corners.cpp:83-120) -- Sobel / Scharr with the scale folded into
  the smoothing kernel (cudafilters/src/filtering.cpp:524-550), row pass then column pass with the border on source
  coordinates, then the blockSize x blockSize sums reading Dx / Dy through the border rule again
  (cuda/corners.cu), then the Harris or min-eigenvalue formula.  Borders follow cudev's rules.
- candidates(): findCorners (cuda/gftt.cu:55-88) with the threshold float(double(max) * qualityLevel), the maximum taken
  over the whole image without the mask (gftt.cpp:120); ordered by response, then raster index, both descending, and
  cut to max(1000, int(0.05 * area)).
- select_sequential(): the reference's minDistance grid loop (gftt.cpp:147-206), written literally.
"""
from __future__ import annotations

import numpy as np

BORDER_REPLICATE, BORDER_REFLECT, BORDER_REFLECT101 = 1, 2, 4
F32 = np.float32


def border_index(i, n: int, border: int) -> np.ndarray:
    """cudev's idx_low(idx_high(i)) (cudev/ptr2d/extrapolation.hpp) for an int array i and a length n >= 1."""
    i = np.asarray(i, dtype=np.int64)
    last = n - 1
    if border == BORDER_REPLICATE:
        return np.clip(i, 0, last)
    if border == BORDER_REFLECT:
        hi = last - np.abs(last - i) + (i > last)
        return (np.abs(hi) - (hi < 0)) % n
    if border == BORDER_REFLECT101:
        hi = np.abs(last - np.abs(last - i)) % n
        return np.abs(hi) % n
    raise ValueError(border)


def sobel_kernel(order: int, ksize: int) -> list:
    """getDerivKernels(..., normalize=false) integer taps: Sobel for ksize > 0, Scharr for ksize <= 0."""
    if ksize <= 0:
        return [-1, 0, 1] if order else [3, 10, 3]
    if ksize == 1 and order > 0:
        ksize = 3
    if ksize == 1:
        return [1]
    if ksize == 3:
        return [-1, 0, 1] if order == 1 else [1, 2, 1]
    k = [1] + [0] * ksize
    for _ in range(ksize - order - 1):
        old = k[0]
        for j in range(1, ksize + 1):
            new = k[j] + k[j - 1]
            k[j - 1] = old
            old = new
    for _ in range(order):
        old = -k[0]
        for j in range(1, ksize + 1):
            new = k[j - 1] - k[j]
            k[j - 1] = old
            old = new
    return k[:ksize]


def deriv_taps(ksize: int, block_size: int, u8: bool):
    """(dx_row, dx_col, dy_row, dy_col) float32 taps: CornerBase's scale (double), multiplied in float into the smoothing
    kernel (kx of d/dy, ky of d/dx)."""
    scale = float(1 << ((ksize if ksize > 0 else 3) - 1)) * block_size
    if ksize < 0:
        scale *= 2.0
    if u8:
        scale *= 255.0
    scale = 1.0 / scale
    d = np.array(sobel_kernel(1, ksize), dtype=F32)
    s = np.array(sobel_kernel(0, ksize), dtype=F32) * F32(scale)
    return d, s, s, d


def _row_pass(src: np.ndarray, taps: np.ndarray, border: int) -> np.ndarray:
    rows, cols = src.shape
    out = np.zeros_like(src)
    x = np.arange(cols)
    for t, w in enumerate(taps):
        out = out + src[:, border_index(x + t - len(taps) // 2, cols, border)] * F32(w)
    return out


def _col_pass(buf: np.ndarray, taps: np.ndarray, border: int) -> np.ndarray:
    rows, cols = buf.shape
    out = np.zeros_like(buf)
    y = np.arange(rows)
    for t, w in enumerate(taps):
        out = out + buf[border_index(y + t - len(taps) // 2, rows, border), :] * F32(w)
    return out


def derivatives(src: np.ndarray, ksize: int, block_size: int, border: int):
    u8 = src.dtype == np.uint8
    img = src.astype(F32)
    dx_row, dx_col, dy_row, dy_col = deriv_taps(ksize, block_size, u8)
    dx = _col_pass(_row_pass(img, dx_row, border), dx_col, border)
    dy = _col_pass(_row_pass(img, dy_row, border), dy_col, border)
    return dx, dy


def response(src: np.ndarray, block_size: int, ksize: int, border: int = BORDER_REFLECT101, harris: bool = False,
             k: float = 0.04) -> np.ndarray:
    """cv::cuda::createHarrisCorner / createMinEigenValCorner(...)->compute(src) for an 8UC1 or 32FC1 image."""
    assert src.ndim == 2 and src.dtype in (np.uint8, np.float32)
    dx, dy = derivatives(src, ksize, block_size, border)
    rows, cols = src.shape
    y, x = np.arange(rows), np.arange(cols)
    a = np.zeros((rows, cols), F32)
    b = np.zeros((rows, cols), F32)
    c = np.zeros((rows, cols), F32)
    h0 = block_size // 2
    for i in range(block_size):
        ry = border_index(y - h0 + i, rows, border)
        for j in range(block_size):
            cx = border_index(x - h0 + j, cols, border)
            ex = dx[ry][:, cx]
            ey = dy[ry][:, cx]
            a = a + ex * ex
            b = b + ex * ey
            c = c + ey * ey
    if harris:
        kf = F32(k)
        return a * c - b * b - kf * (a + c) * (a + c)
    a = a * F32(0.5)
    c = c * F32(0.5)
    return (a + c) - np.sqrt((a - c) * (a - c) + b * b)


def keep_capacity(rows: int, cols: int) -> int:
    return max(1000, int(rows * cols * 0.05))


def candidates(eig: np.ndarray, quality: float, mask: np.ndarray | None = None):
    """Candidate positions (N, 2) int in the detector's order, and the count before the capacity cut."""
    rows, cols = eig.shape
    thr = F32(float(eig.max()) * quality)
    ok = np.zeros((rows, cols), bool)
    if rows >= 3 and cols >= 3:
        v = eig[1:-1, 1:-1]
        m = v.copy()
        for oy in (-1, 0, 1):
            for ox in (-1, 0, 1):
                if oy or ox:
                    m = np.fmax(eig[1 + oy:rows - 1 + oy, 1 + ox:cols - 1 + ox], m)
        ok[1:-1, 1:-1] = (v > thr) & (v == m)
    if mask is not None:
        ok &= mask != 0
    ys, xs = np.nonzero(ok)
    vals = eig[ys, xs]
    idx = ys.astype(np.int64) * cols + xs
    order = np.lexsort((-idx, -vals.astype(np.float64)))  # response descending, then raster index descending
    n = len(order)
    order = order[:keep_capacity(rows, cols)]
    return np.stack([xs[order], ys[order]], axis=1), n


def cv_round(v: float) -> int:
    return int(np.rint(v))  # half to even, as cvRound


def select_sequential(pts: np.ndarray, min_distance: float, max_corners: int, rows: int, cols: int) -> np.ndarray:
    """gftt.cpp:147-206, line for line."""
    tmp2 = []
    cell_size = cv_round(min_distance)
    grid_width = (cols + cell_size - 1) // cell_size
    grid_height = (rows + cell_size - 1) // cell_size
    grid = [[] for _ in range(grid_width * grid_height)]
    md2 = min_distance * min_distance
    for px, py in np.asarray(pts, dtype=F32):
        good = True
        x_cell = int(px / F32(cell_size))
        y_cell = int(py / F32(cell_size))
        x1, y1, x2, y2 = x_cell - 1, y_cell - 1, x_cell + 1, y_cell + 1
        x1, y1 = max(0, x1), max(0, y1)
        x2, y2 = min(grid_width - 1, x2), min(grid_height - 1, y2)
        for yy in range(y1, y2 + 1):
            for xx in range(x1, x2 + 1):
                for mx, my in grid[yy * grid_width + xx]:
                    dx = px - mx
                    dy = py - my
                    if float(dx * dx + dy * dy) < md2:
                        good = False
                        break
                if not good:
                    break
            if not good:
                break
        if good:
            grid[y_cell * grid_width + x_cell].append((px, py))
            tmp2.append((px, py))
            if max_corners > 0 and len(tmp2) == max_corners:
                break
    return np.array(tmp2, dtype=F32).reshape(-1, 2)


def selection_rounds(pts: np.ndarray, min_distance: float, rows: int, cols: int) -> int:
    """Rounds the engine's parallel greedy selection takes over the kept candidates `pts` (priority order): in each round
    an undecided candidate is rejected when a higher-priority conflicting candidate was accepted in an EARLIER round,
    accepted when all of them were rejected in earlier rounds, else it waits.  The decided sets equal the sequential
    loop's; this counts the rounds until none is undecided (1 when there is no candidate)."""
    cell = cv_round(min_distance)
    md2 = min_distance * min_distance
    reach = int(np.floor(min_distance))
    owner = {}
    d = np.zeros(len(pts), np.int64)
    acc = np.zeros(len(pts), bool)
    for i, (px, py) in enumerate(np.asarray(pts, dtype=np.int64)):
        xc, yc = int(F32(px) / F32(cell)), int(F32(py) / F32(cell))
        ra, rall = None, 0
        for qy in range(max(py - reach, max(0, yc - 1) * cell), min(py + reach, (yc + 2) * cell - 1, rows - 1) + 1):
            for qx in range(max(px - reach, max(0, xc - 1) * cell), min(px + reach, (xc + 2) * cell - 1, cols - 1) + 1):
                j = owner.get((qx, qy))
                if j is None:
                    continue
                dx, dy = F32(px) - F32(qx), F32(py) - F32(qy)
                if float(dx * dx + dy * dy) < md2:
                    rall = max(rall, d[j] + 1)
                    if acc[j]:
                        ra = d[j] + 1 if ra is None else min(ra, d[j] + 1)
        d[i], acc[i] = (ra, False) if ra is not None else (rall, True)
        owner[(int(px), int(py))] = i
    return int(d.max()) + 1 if len(pts) else 1


def gftt(image: np.ndarray, max_corners: int = 1000, quality_level: float = 0.01, min_distance: float = 0.0,
         block_size: int = 3, use_harris: bool = False, harris_k: float = 0.04, mask: np.ndarray | None = None):
    """cv::cuda::createGoodFeaturesToTrackDetector(...)->detect(image, corners, mask): (N, 2) float32 corners and the
    candidate count before the capacity cut."""
    eig = response(image, block_size, 3, BORDER_REFLECT101, use_harris, harris_k)
    pts, n = candidates(eig, quality_level, mask)
    rows, cols = image.shape
    if min_distance < 1:
        m = min(max_corners, len(pts)) if max_corners > 0 else len(pts)
        return pts[:m].astype(F32), n
    return select_sequential(pts, min_distance, max_corners, rows, cols), n
