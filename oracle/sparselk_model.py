"""numpy model of the reference's sparse pyramidal Lucas-Kanade, ``cv::cuda::SparsePyrLKOpticalFlow``
(modules/cudaoptflow/src/pyrlk.cpp:153-236 + src/cuda/pyrlk.cu sparseKernel / sparseKernel_), restated with the
engine's own float32 arithmetic (opencv_contrib_b200/csrc/sparselk.cu, built with -fmad=false so that every operator
rounds once) so that the two agree bit for bit.

TEST INFRASTRUCTURE (see oracle/__init__.py).  The engine's documented choices, restated:

* input: deinterleaved to float planes; the pyramid is pyrDown (``denselk_model.pyr_down``, the engine's pyr_tap5
  chain), rounded to the element type with rint(clamp(lo, hi)) for integer depths (8-bit included);
* texture path (8UC1, 8UC4, 16UC4, 32FC1, 32FC4): bilinear with 8-bit weights floor(frac * 256 + 0.5) / 256,
  clamped addresses, integer texels divided by 255 or 65535 (correctly rounded);
* software path (every 3-channel type, 16UC1, 32SC1, 32SC4): exact weights from floor(x), zero outside the image,
  the coordinate clamped to [-4, n + 4], the result rounded to the element type for integer depths;
* reductions: one 256-thread block per point; element e belongs to thread e % 256, which sums its elements in order
  of e and, within an element, in order of channel; each warp reduces with shfl_down 16 / 8 / 4 / 2 / 1 and the 8
  warp sums are added in order (``block_sum``);
* control flow as the kernels: a point outside the level, a singular matrix (D < FLT_EPSILON) or a track that leaves
  the level during the iterations returns without writing nextPts, and clears status only on level 0; the iterations
  stop when |dx| < 0.01 and |dy| < 0.01; err is written only when level 0 completes, as
  sum |J - I| / (min(cn, 3) * w * h) * scale, scale 255 for 8-bit images on the texture path and 1 otherwise.

``calc(..., counters=list)`` appends one ``Counters`` per level, coarsest first, so that a test can prove that its
input takes the branches it is there for.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .denselk_model import _blend, pyr_down

F = np.float32
SB = 256  # threads per point
FLT_EPSILON = F(np.finfo(np.float32).eps)
COUNTER_NAMES = ("outside_prev", "singular", "left_during_iters", "converged", "hit_iters")
DEPTHS = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 2, np.dtype(np.int32): 4, np.dtype(np.float32): 5}
RANGES = {0: (0.0, 255.0), 2: (0.0, 65535.0), 4: (-2147483648.0, 2147483520.0)}  # saturate_cast range, as float


@dataclass
class Counters:
    """Per-level point counts.  outside_prev: prevPt / 2^level outside the level (returns first); singular:
    D < FLT_EPSILON; left_during_iters: the track left the level before an iteration; converged: the step fell
    below 0.01 in both axes; hit_iters: ran all ``iters`` iterations (every point that got that far when iters is 0)."""
    outside_prev: int = 0
    singular: int = 0
    left_during_iters: int = 0
    converged: int = 0
    hit_iters: int = 0

    def as_tuple(self):
        return tuple(int(getattr(self, k)) for k in COUNTER_NAMES)


def is_soft(depth: int, cn: int) -> bool:
    """The reference's sparse_caller specialisations: which (depth, cn) run the software sampler."""
    return cn == 3 or (depth == 2 and cn == 1) or depth == 4


def _quantize(p, depth):
    if depth == 5:
        return p
    lo, hi = RANGES[depth]
    return np.rint(np.minimum(np.maximum(p, F(lo)), F(hi))).astype(F)


def pyramid(img: np.ndarray, max_level: int):
    """Levels as (cn, rows, cols) float32: the deinterleaved input, then pyrDown rounded to the element type."""
    depth = DEPTHS[img.dtype]
    planes = img[None] if img.ndim == 2 else np.moveaxis(img, -1, 0)
    levels = [planes.astype(F)]
    for _ in range(max_level):
        levels.append(np.stack([_quantize(pyr_down(p), depth) for p in levels[-1]]))
    return levels


def tex_axis(coord, n):
    """Texture addressing along one axis: clamped lower / upper texel index and the 8-bit weight of the upper one."""
    b = (coord - F(0.5)).astype(F)
    f = np.floor(b)
    a = (np.floor(((b - f) * F(256)).astype(F) + F(0.5)) * F(1 / 256)).astype(F)
    i0 = np.minimum(np.maximum(f, F(-2)), F(n + 1)).astype(np.int64)
    return np.clip(i0, 0, n - 1), np.clip(i0 + 1, 0, n - 1), a


def sample_tex(planes, y, x, norm):
    """k_sparse_lk sp_tex / k_sparse_lk_mc SAMP_TEX for every plane: (cn,) + x.shape."""
    _, rows, cols = planes.shape
    xa, xc, ax = tex_axis(x, cols)
    ya, yc, ay = tex_axis(y, rows)
    out = []
    for p in planes:
        t = [p[ya, xa], p[ya, xc], p[yc, xa], p[yc, xc]]
        if norm != 1:
            t = [(v / F(norm)).astype(F) for v in t]
        out.append(_blend(ax, ay, *t))
    return np.stack(out)


def sample_soft(planes, y, x, depth):
    """k_sparse_lk_mc SAMP_SOFT (LinearFilter<BorderReader<BrdConstant>> + saturate_cast): (cn,) + x.shape."""
    _, rows, cols = planes.shape
    fx = np.floor(np.minimum(np.maximum(x, F(-4)), F(cols + 4)))
    fy = np.floor(np.minimum(np.maximum(y, F(-4)), F(rows + 4)))
    x1, y1 = fx.astype(np.int64), fy.astype(np.int64)
    x2, y2 = x1 + 1, y1 + 1
    x1f, x2f, y1f, y2f = (v.astype(F) for v in (x1, x2, y1, y2))
    w11 = ((x2f - x).astype(F) * (y2f - y).astype(F)).astype(F)
    w12 = ((x - x1f).astype(F) * (y2f - y).astype(F)).astype(F)
    w21 = ((x2f - x).astype(F) * (y - y1f).astype(F)).astype(F)
    w22 = ((x - x1f).astype(F) * (y - y1f).astype(F)).astype(F)
    r1, r2 = (y1 >= 0) & (y1 < rows), (y2 >= 0) & (y2 < rows)
    c1, c2 = (x1 >= 0) & (x1 < cols), (x2 >= 0) & (x2 < cols)
    cy1, cy2 = np.clip(y1, 0, rows - 1), np.clip(y2, 0, rows - 1)
    cx1, cx2 = np.clip(x1, 0, cols - 1), np.clip(x2, 0, cols - 1)
    out = []
    for p in planes:
        o = np.zeros(x.shape, F)
        for ok, yy, xx, w in ((r1 & c1, cy1, cx1, w11), (r1 & c2, cy1, cx2, w12),
                              (r2 & c1, cy2, cx1, w21), (r2 & c2, cy2, cx2, w22)):
            o = (o + (np.where(ok, p[yy, xx], F(0)) * w).astype(F)).astype(F)
        out.append(_quantize(o, depth))
    return np.stack(out)


def block_sum(v):
    """block_sum of sparselk.cu for every point: v is (points, elements, channels) float32 in the kernel's element
    order; returns (points,) float32."""
    P, E, C = v.shape
    acc = np.zeros((P, SB), F)
    for r in range(0, E, SB):
        n = min(SB, E - r)
        for c in range(C):
            acc[:, :n] = (acc[:, :n] + v[:, r:r + n, c]).astype(F)  # thread t: elements t, t + 256, ... in order
    w = acc.reshape(P, SB // 32, 32)
    for o in (16, 8, 4, 2, 1):  # __shfl_down_sync tree: lane 0 of each warp
        w = (w[..., :o] + w[..., o:2 * o]).astype(F)
    w = w[..., 0]
    s = w[:, 0]
    for k in range(1, SB // 32):
        s = (s + w[:, k]).astype(F)
    return s


def _scharr(s):
    """3 a + 10 b + 3 c - (3 d + 10 e + 3 f), left to right, each product and sum rounded."""
    a, b, c, d, e, f = s
    p = (((F(3) * a).astype(F) + (F(10) * b).astype(F)).astype(F) + (F(3) * c).astype(F)).astype(F)
    m = (((F(3) * d).astype(F) + (F(10) * e).astype(F)).astype(F) + (F(3) * f).astype(F)).astype(F)
    return (p - m).astype(F)


def _cells(v):
    """(cn, points, elements) -> (points, elements, cn): the kernels' per-thread order (element, then channel)."""
    return np.moveaxis(v, 0, -1)


def calc(I0: np.ndarray, I1: np.ndarray, prev_pts: np.ndarray, win_size=(21, 21), max_level=3, iters=30,
         next_pts=None, want_err=True, counters=None):
    """SparsePyrLKOpticalFlowImpl::calc.  I0 / I1: (rows, cols) or (rows, cols, cn) uint8 / uint16 / int32 / float32;
    prev_pts (N, 2) float32; next_pts: the caller's estimate (use_initial_flow) or None.  Returns (nextPts, status,
    err): nextPts (N, 2) float32 including the stale values of points that returned early, status uint8, err float32
    with NaN where the engine does not write it (every point when want_err is False)."""
    assert I0.dtype == I1.dtype and I0.shape == I1.shape
    depth = DEPTHS[I0.dtype]
    cn = 1 if I0.ndim == 2 else I0.shape[2]
    assert cn in (1, 3, 4)
    soft = is_soft(depth, cn)
    norm = 1.0 if soft or depth == 5 else (255.0 if depth == 0 else 65535.0)
    err_scale = F(255) if (not soft and depth == 0) else F(1)
    win_x, win_y = win_size
    half_x, half_y = (win_x - 1) // 2, (win_y - 1) // 2
    n_win = win_x * win_y
    pI, pJ = pyramid(I0, max_level), pyramid(I1, max_level)

    def sample(planes, y, x):
        return sample_soft(planes, y, x, depth) if soft else sample_tex(planes, y, x, norm)

    prev = np.asarray(prev_pts, F).reshape(-1, 2)
    n = len(prev)
    scale = F(1.0 / (1 << max_level) / 2.0)
    src = prev if next_pts is None else np.asarray(next_pts, F).reshape(-1, 2)
    nxt = (src * scale).astype(F)  # k_sparse_init
    status = np.ones(n, np.uint8)
    err = np.full(n, np.nan, F)
    e = np.arange(n_win)
    yB, xB = (e // win_x).astype(F)[None, :], (e % win_x).astype(F)[None, :]

    for level in range(max_level, -1, -1):
        cnt = Counters()
        I, J = pI[level], pJ[level]
        _, rows, cols = I.shape
        inv = F(1) / F(1 << level)
        px, py = (prev[:, 0] * inv).astype(F), (prev[:, 1] * inv).astype(F)
        outside = (px < 0) | (px >= F(cols)) | (py < 0) | (py >= F(rows))
        cnt.outside_prev = int(outside.sum())
        if level == 0:
            status[outside] = 0
        k = np.nonzero(~outside)[0]
        px, py = (px[k] - F(half_x)).astype(F), (py[k] - F(half_y)).astype(F)
        x = ((px[:, None] + xB).astype(F) + F(0.5)).astype(F)
        y = ((py[:, None] + yB).astype(F) + F(0.5)).astype(F)
        xm, xp = (x - F(1)).astype(F), (x + F(1)).astype(F)
        ym, yp = (y - F(1)).astype(F), (y + F(1)).astype(F)
        Ip = sample(I, y, x)
        mm, m0, mp = sample(I, ym, xm), sample(I, ym, x), sample(I, ym, xp)
        zm, zp = sample(I, y, xm), sample(I, y, xp)
        pm, p0, pp = sample(I, yp, xm), sample(I, yp, x), sample(I, yp, xp)
        dIdx = _scharr((mp, zp, pp, mm, zm, pm))
        dIdy = _scharr((pm, p0, pp, mm, m0, mp))
        del mm, m0, mp, zm, zp, pm, p0, pp
        A11 = block_sum(_cells((dIdx * dIdx).astype(F)))
        A12 = block_sum(_cells((dIdx * dIdy).astype(F)))
        A22 = block_sum(_cells((dIdy * dIdy).astype(F)))
        D = ((A11 * A22).astype(F) - (A12 * A12).astype(F)).astype(F)
        sing = D < FLT_EPSILON
        cnt.singular = int(sing.sum())
        if level == 0:
            status[k[sing]] = 0
        keep = ~sing
        k, Ip, dIdx, dIdy = k[keep], Ip[:, keep], dIdx[:, keep], dIdy[:, keep]
        D = (F(1) / D[keep]).astype(F)
        A11, A12, A22 = (A11[keep] * D).astype(F), (A12[keep] * D).astype(F), (A22[keep] * D).astype(F)
        nx = ((nxt[k, 0] * F(2)).astype(F) - F(half_x)).astype(F)
        ny = ((nxt[k, 1] * F(2)).astype(F) - F(half_y)).astype(F)
        active = np.ones(len(k), bool)   # still iterating
        alive = np.ones(len(k), bool)    # will write nextPts
        for _ in range(iters):
            left = active & ((nx < F(-half_x)) | (nx >= F(cols)) | (ny < F(-half_y)) | (ny >= F(rows)))
            alive &= ~left
            active &= ~left
            a = np.nonzero(active)[0]
            if len(a) == 0:
                break
            Jv = sample(J, ((ny[a, None] + yB).astype(F) + F(0.5)).astype(F), ((nx[a, None] + xB).astype(F) + F(0.5)).astype(F))
            diff = ((Jv - Ip[:, a]).astype(F) * F(32)).astype(F)
            b0 = block_sum(_cells((diff * dIdx[:, a]).astype(F)))
            b1 = block_sum(_cells((diff * dIdy[:, a]).astype(F)))
            dx = ((A12[a] * b1).astype(F) - (A22[a] * b0).astype(F)).astype(F)
            dy = ((A12[a] * b0).astype(F) - (A11[a] * b1).astype(F)).astype(F)
            nx[a] = (nx[a] + dx).astype(F)
            ny[a] = (ny[a] + dy).astype(F)
            conv = (np.abs(dx) < F(0.01)) & (np.abs(dy) < F(0.01))
            cnt.converged += int(conv.sum())
            active[a[conv]] = False
        cnt.left_during_iters = int((~alive).sum())
        cnt.hit_iters = int((alive & active).sum())
        if level == 0:
            status[k[~alive]] = 0
            if want_err:
                w = np.nonzero(alive)[0]
                Jv = sample(J, ((ny[w, None] + yB).astype(F) + F(0.5)).astype(F), ((nx[w, None] + xB).astype(F) + F(0.5)).astype(F))
                ev = block_sum(_cells(np.abs((Jv - Ip[:, w]).astype(F))))
                err[k[w]] = ((ev / F(min(cn, 3) * n_win)).astype(F) * err_scale).astype(F)
        w = k[alive]
        nxt[w, 0] = (nx[alive] + F(half_x)).astype(F)
        nxt[w, 1] = (ny[alive] + F(half_y)).astype(F)
        if counters is not None:
            counters.append(cnt)
    return nxt, status, err
