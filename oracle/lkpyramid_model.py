"""The video module's pyramidal Lucas-Kanade tracker (cv::calcOpticalFlowPyrLK, cv::buildOpticalFlowPyramid) restated in
numpy with cv2's own types: uint8 levels, int16 Scharr derivatives, int32 fixed-point bilinear taps and float32 sums.

The float sums follow the order cv2 4.13's x86 build adds them (128-bit universal intrinsics, SSE baseline):

  * covariance A: per window row, elements in chunks of 8 (x <= W*cn - 8) go to 4 float lanes, lane k taking element
    x + k and then x + k + 4, each lane a sequential float sum over rows and chunks; the elements left over in each row go to one scalar
    float sum, row-major.  A = scalar + ((lane0 + lane2) + (lane1 + lane3)) -- the movehl-then-add lane reduction;
  * mismatch b: per row, chunks of 8 elements; int32 pair sums It_k Ix_k + It_{k+4} Ix_{k+4} (k = 0..3) are converted
    to float and added to two 4-lane accumulators, [b1(0,4), b2(0,4), b1(1,5), b2(1,5)] and the same for (2,6), (3,7);
    the leftover elements go to a scalar sum.  b1 = scalar + ((q0[0] + q1[0]) + (q0[2] + q1[2])), b2 likewise with
    lanes 1 and 3;
  * the error: a sequential float sum of |diff| in row-major order, divided by 32 W cn H.

``LANE_REDUCE`` and the chunk widths are the choices tests/test_lkpyramid_model_cpu.py pins against the live cv2.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

W_BITS = 14
FLT_SCALE = np.float32(1.0 / (1 << 20))
FLT_EPSILON = np.float32(np.finfo(np.float32).eps)
OPTFLOW_USE_INITIAL_FLOW = 4
OPTFLOW_LK_GET_MIN_EIGENVALS = 8
COUNT, EPS = 1, 2
BORDER_CONSTANT, BORDER_REFLECT_101, BORDER_ISOLATED = 0, 4, 16

A_CHUNK = 8
B_CHUNK = 8
LANE_REDUCE = "movehl"  # ((l0 + l2) + (l1 + l3)); "hadd" would be ((l0 + l1) + (l2 + l3))

f32 = np.float32


def reflect101(p, n):
    """cv::borderInterpolate(p, n, BORDER_REFLECT_101), vectorised."""
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


def _as3(img):
    img = np.asarray(img)
    return img[..., None] if img.ndim == 2 else img


def pyr_down(img, dsize):
    """cv::pyrDown for 8U: 5x5 [1 4 6 4 1]^2 / 256 with (s + 128) >> 8, BORDER_REFLECT_101 of the source."""
    src = _as3(img).astype(np.int32)
    h, w, _ = src.shape
    dw, dh = dsize
    k = np.array([1, 4, 6, 4, 1], np.int32)
    cols = reflect101(2 * np.arange(dw)[:, None] + np.arange(-2, 3)[None, :], w)  # (dw, 5)
    rows = reflect101(2 * np.arange(dh)[:, None] + np.arange(-2, 3)[None, :], h)
    hsum = np.einsum("ywkc,k->ywc", src[:, cols, :], k)  # (h, dw, cn)
    vsum = np.einsum("ykwc,k->ywc", hsum[rows], k)
    return ((vsum + 128) >> 8).astype(np.uint8)


def scharr_deriv(img):
    """calcSharrDeriv: int16 (rows, cols, 2 cn), per channel (Ix, Iy); one-pixel reflect-101 rows and columns."""
    src = _as3(img).astype(np.int32)
    h, w, cn = src.shape
    ym = reflect101(np.arange(h) - 1, h)
    yp = reflect101(np.arange(h) + 1, h)
    t0 = (src[ym] + src[yp]) * 3 + src * 10
    t1 = src[yp] - src[ym]
    xm = reflect101(np.arange(w) - 1, w)
    xp = reflect101(np.arange(w) + 1, w)
    ix = (t0[:, xp] - t0[:, xm]).astype(np.int16)
    iy = ((t1[:, xp] + t1[:, xm]) * 3 + t1 * 10).astype(np.int16)
    out = np.empty((h, w, 2 * cn), np.int16)
    out[..., 0::2] = ix
    out[..., 1::2] = iy
    return out


def pad(a, bw, bh, mode):
    a = _as3(a)
    h, w = a.shape[:2]
    if mode == BORDER_CONSTANT:
        out = np.zeros((h + 2 * bh, w + 2 * bw, a.shape[2]), a.dtype)
        out[bh:bh + h, bw:bw + w] = a
        return out
    ry = reflect101(np.arange(-bh, h + bh), h)
    rx = reflect101(np.arange(-bw, w + bw), w)
    return a[ry][:, rx]


@dataclass
class Pyramid:
    """buildOpticalFlowPyramid's output: padded levels (border win), optional padded derivatives."""
    win: tuple
    levels: list = field(default_factory=list)   # padded uint8 (h + 2 bh, w + 2 bw, cn)
    derivs: list = field(default_factory=list)   # padded int16 (h + 2 bh, w + 2 bw, 2 cn), or empty

    @property
    def max_level(self):
        return len(self.levels) - 1

    def interior(self, lvl, deriv=False):
        bw, bh = self.win
        a = (self.derivs if deriv else self.levels)[lvl]
        return a[bh:a.shape[0] - bh, bw:a.shape[1] - bw]


def build_pyramid(img, win_size, max_level, with_derivatives=True, pyr_border=BORDER_REFLECT_101,
                  deriv_border=BORDER_CONSTANT):
    """cv::buildOpticalFlowPyramid; returns (max level built, Pyramid)."""
    img = _as3(img)
    bw, bh = int(win_size[0]), int(win_size[1])
    assert img.dtype == np.uint8 and bw > 2 and bh > 2
    P = Pyramid((bw, bh))
    this = img
    h, w = img.shape[:2]
    for level in range(max_level + 1):
        if level:
            this = pyr_down(this, (w, h))
        P.levels.append(pad(this, bw, bh, pyr_border & ~BORDER_ISOLATED))
        if with_derivatives:
            P.derivs.append(pad(scharr_deriv(this), bw, bh, deriv_border & ~BORDER_ISOLATED))
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= bw or h <= bh:
            return level, P
    return max_level, P


def _reduce(q):
    if LANE_REDUCE == "hadd":
        return (q[:, 0] + q[:, 1]) + (q[:, 2] + q[:, 3])
    return (q[:, 0] + q[:, 2]) + (q[:, 1] + q[:, 3])


def _weights(a, b):
    one = f32(1)
    s = f32(1 << W_BITS)
    iw00 = np.rint((one - a) * (one - b) * s).astype(np.int32)
    iw01 = np.rint(a * (one - b) * s).astype(np.int32)
    iw10 = np.rint((one - a) * b * s).astype(np.int32)
    iw11 = (1 << W_BITS) - iw00 - iw01 - iw10
    return iw00, iw01, iw10, iw11


def _cv_floor(v):
    """cvFloor with x86's integer-indefinite result for NaN and out-of-range values."""
    out = np.full(v.shape, np.iinfo(np.int32).min, np.int64)
    ok = np.isfinite(v) & (v >= -2147483648.0) & (v < 2147483648.0)
    out[ok] = np.floor(v[ok]).astype(np.int64)
    return out


def _gather(padded, iy, ix, bw, bh, win, ncomp):
    """(N, wh + 1, (ww + 1) * ncomp) block of the padded level whose top-left pixel is (iy, ix) in interior coords."""
    ww, wh = win
    flat = padded.reshape(padded.shape[0], -1)
    rows = (iy + bh)[:, None] + np.arange(wh + 1)[None, :]
    cols = ((ix + bw) * ncomp)[:, None] + np.arange((ww + 1) * ncomp)[None, :]
    return flat[rows[:, :, None], cols[:, None, :]].astype(np.int32)


def _interp(block, w, ncomp, bits, win):
    ww, wh = win
    n = ww * ncomp
    w00, w01, w10, w11 = (x[:, None, None] for x in w)
    s = (block[:, :wh, :n] * w00 + block[:, :wh, ncomp:ncomp + n] * w01 +
         block[:, 1:, :n] * w10 + block[:, 1:, ncomp:ncomp + n] * w11)
    return (s + (1 << (bits - 1))) >> bits


def calc(prev, nxt, prev_pts, next_pts=None, win_size=(21, 21), max_level=3, criteria=(COUNT | EPS, 30, 0.01),
         flags=0, min_eig_threshold=1e-4, counters=None):
    """cv::calcOpticalFlowPyrLK.  prev / nxt: uint8 images (H, W[, cn]) or Pyramid objects.  Returns (nextPts (N, 2)
    float32, status (N,) uint8, err (N,) float32, written (N,) bool: where cv2 writes err)."""
    ww, wh = int(win_size[0]), int(win_size[1])
    assert max_level >= 0 and ww > 2 and wh > 2
    pts = np.asarray(prev_pts, np.float32).reshape(-1, 2)
    npts = len(pts)
    ctype, maxc, eps = criteria
    maxc = 30 if not (ctype & COUNT) else min(max(int(maxc), 0), 100)
    eps = 0.01 if not (ctype & EPS) else min(max(float(eps), 0.0), 10.0)
    eps *= eps
    if counters is None:
        counters = {}
    for k in ("out_of_image", "rejected_mineig", "rejected_det", "out_of_window", "eps_stop", "half_step", "err_out"):
        counters.setdefault(k, 0)

    if isinstance(prev, Pyramid):
        assert prev.win[0] >= ww and prev.win[1] >= wh
        max_level = min(max_level, prev.max_level)
    if isinstance(nxt, Pyramid):
        assert nxt.win[0] >= ww and nxt.win[1] >= wh
        max_level = min(max_level, nxt.max_level)
    if not isinstance(prev, Pyramid):
        max_level, prev = build_pyramid(prev, (ww, wh), max_level, True)
    if not isinstance(nxt, Pyramid):
        max_level, nxt = build_pyramid(nxt, (ww, wh), max_level, False)

    status = np.ones(npts, np.uint8)
    err = np.zeros(npts, np.float32)
    written = np.zeros(npts, bool)
    out = np.empty((npts, 2), np.float32) if next_pts is None else np.asarray(next_pts, np.float32).reshape(-1, 2).copy()
    if npts == 0:
        return out, status, err, written
    half = np.array([(ww - 1) * 0.5, (wh - 1) * 0.5], np.float32)
    want_mineig = bool(flags & OPTFLOW_LK_GET_MIN_EIGENVALS)

    for level in range(max_level, -1, -1):
        I = prev.levels[level]
        cn = I.shape[2]
        if prev.derivs:
            dI = prev.derivs[level]
            dbw, dbh = prev.win
        else:
            dI = pad(scharr_deriv(prev.interior(level)), ww, wh, BORDER_CONSTANT)
            dbw, dbh = ww, wh
        J = nxt.levels[level]
        rows, cols = I.shape[0] - 2 * prev.win[1], I.shape[1] - 2 * prev.win[0]
        assert (J.shape[0] - 2 * nxt.win[1], J.shape[1] - 2 * nxt.win[0]) == (rows, cols) and J.shape[2] == cn
        n = ww * cn

        pp = pts * f32(1.0 / (1 << level))
        if level == max_level:
            nx = out * f32(1.0 / (1 << level)) if flags & OPTFLOW_USE_INITIAL_FLOW else pp.copy()
        else:
            nx = out * f32(2)
        out = nx.copy()
        pp = pp - half
        ipx, ipy = _cv_floor(pp[:, 0]), _cv_floor(pp[:, 1])
        inside = (ipx >= -ww) & (ipx < cols) & (ipy >= -wh) & (ipy < rows)
        if level == 0:
            status[~inside] = 0
            err[~inside] = 0
            written[~inside] = True
        counters["out_of_image"] += int((~inside).sum())
        idx = np.nonzero(inside)[0]
        if len(idx) == 0:
            continue
        ipx, ipy, pp = ipx[idx], ipy[idx], pp[idx]
        a = pp[:, 0] - ipx.astype(np.float32)
        b = pp[:, 1] - ipy.astype(np.float32)
        w = _weights(a, b)
        Iw = _interp(_gather(I, ipy, ipx, prev.win[0], prev.win[1], (ww, wh), cn), w, cn, W_BITS - 5, (ww, wh))
        dblk = _gather(dI, ipy, ipx, dbw, dbh, (ww, wh), 2 * cn)
        dW = _interp(dblk, w, 2 * cn, W_BITS, (ww, wh))  # (m, wh, 2 n): Ix, Iy interleaved
        Ix, Iy = dW[:, :, 0::2], dW[:, :, 1::2]
        m = len(idx)

        # covariance: 4-lane chunks + scalar tail
        qA = [np.zeros((m, 4), np.float32) for _ in range(3)]
        iA = [np.zeros(m, np.float32) for _ in range(3)]
        nch = (n // A_CHUNK) * A_CHUNK if n >= A_CHUNK else 0
        fx_all, fy_all = Ix.astype(np.float32), Iy.astype(np.float32)
        for y in range(wh):
            for x0 in range(0, nch, A_CHUNK):
                for L in range(A_CHUNK):
                    fx, fy = fx_all[:, y, x0 + L], fy_all[:, y, x0 + L]
                    lane = L % 4
                    qA[2][:, lane] += fy * fy
                    qA[1][:, lane] += fx * fy
                    qA[0][:, lane] += fx * fx
            for x in range(nch, n):
                ix, iy = Ix[:, y, x], Iy[:, y, x]
                iA[0] += (ix * ix).astype(np.float32)
                iA[1] += (ix * iy).astype(np.float32)
                iA[2] += (iy * iy).astype(np.float32)
        A11, A12, A22 = ((iA[k] + _reduce(qA[k])) * FLT_SCALE for k in range(3))
        D = A11 * A22 - A12 * A12
        minEig = ((A22 + A11) - np.sqrt((A11 - A22) * (A11 - A22) + f32(4) * A12 * A12)) / f32(2 * ww * wh)
        if want_mineig:
            err[idx] = minEig
            written[idx] = True
        bad_eig = minEig < f32(min_eig_threshold)
        bad = bad_eig | (D < FLT_EPSILON)
        counters["rejected_mineig"] += int(bad_eig.sum())
        counters["rejected_det"] += int((~bad_eig & (D < FLT_EPSILON)).sum())
        if level == 0:
            status[idx[bad]] = 0
        keep = ~bad
        idx, Iw, Ix, Iy = idx[keep], Iw[keep], Ix[keep], Iy[keep]
        A11, A12, A22 = A11[keep], A12[keep], A22[keep]
        D = f32(1) / D[keep]
        m = len(idx)
        npt = out[idx] - half
        prev_delta = np.zeros((m, 2), np.float32)
        active = np.ones(m, bool)
        nbch = (n // B_CHUNK) * B_CHUNK
        for j in range(maxc):
            act = np.nonzero(active)[0]
            if len(act) == 0:
                break
            p = npt[act]
            inx, iny = _cv_floor(p[:, 0]), _cv_floor(p[:, 1])
            ok = (inx >= -ww) & (inx < cols) & (iny >= -wh) & (iny < rows)
            gone = act[~ok]
            counters["out_of_window"] += len(gone)
            if level == 0:
                status[idx[gone]] = 0
            active[gone] = False
            act, inx, iny, p = act[ok], inx[ok], iny[ok], p[ok]
            if len(act) == 0:
                break
            a = p[:, 0] - inx.astype(np.float32)
            b = p[:, 1] - iny.astype(np.float32)
            w = _weights(a, b)
            Jw = _interp(_gather(J, iny, inx, nxt.win[0], nxt.win[1], (ww, wh), cn), w, cn, W_BITS - 5, (ww, wh))
            diff = Jw - Iw[act]
            ix_a, iy_a = Ix[act], Iy[act]
            k = len(act)
            q0 = np.zeros((k, 4), np.float32)
            q1 = np.zeros((k, 4), np.float32)
            ib1 = np.zeros(k, np.float32)
            ib2 = np.zeros(k, np.float32)
            for y in range(wh):
                for x0 in range(0, nbch, B_CHUNK):
                    d = diff[:, y, x0:x0 + 8]
                    gx = ix_a[:, y, x0:x0 + 8]
                    gy = iy_a[:, y, x0:x0 + 8]
                    px = (d[:, 0:4] * gx[:, 0:4] + d[:, 4:8] * gx[:, 4:8]).astype(np.float32)
                    py = (d[:, 0:4] * gy[:, 0:4] + d[:, 4:8] * gy[:, 4:8]).astype(np.float32)
                    q0 += np.stack([px[:, 0], py[:, 0], px[:, 1], py[:, 1]], 1)
                    q1 += np.stack([px[:, 2], py[:, 2], px[:, 3], py[:, 3]], 1)
                for x in range(nbch, n):
                    ib1 += (diff[:, y, x] * ix_a[:, y, x]).astype(np.float32)
                    ib2 += (diff[:, y, x] * iy_a[:, y, x]).astype(np.float32)
            s = q0 + q1
            b1 = (ib1 + (s[:, 0] + s[:, 2])) * FLT_SCALE
            b2 = (ib2 + (s[:, 1] + s[:, 3])) * FLT_SCALE
            dx = (A12[act] * b2 - A22[act] * b1) * D[act]
            dy = (A12[act] * b1 - A11[act] * b2) * D[act]
            p = np.stack([p[:, 0] + dx, p[:, 1] + dy], 1)
            npt[act] = p
            out[idx[act]] = p + half
            stop = dx.astype(np.float64) * dx + dy.astype(np.float64) * dy <= eps
            counters["eps_stop"] += int(stop.sum())
            osc = ~stop & (j > 0) & (np.abs(dx + prev_delta[act, 0]) < 0.01) & (np.abs(dy + prev_delta[act, 1]) < 0.01)
            counters["half_step"] += int(osc.sum())
            hs = idx[act[osc]]
            out[hs] = out[hs] - np.stack([dx[osc], dy[osc]], 1) * f32(0.5)
            prev_delta[act] = np.stack([dx, dy], 1)
            active[act[stop | osc]] = False

        if level == 0 and not want_mineig:
            sel = idx[status[idx] != 0]
            if len(sel) == 0:
                continue
            pos = np.nonzero(np.isin(idx, sel))[0]
            p = out[sel] - half
            inx, iny = _cv_floor(p[:, 0]), _cv_floor(p[:, 1])
            ok = (inx >= -ww) & (inx < cols) & (iny >= -wh) & (iny < rows)
            status[sel[~ok]] = 0
            counters["err_out"] += int((~ok).sum())
            sel, pos, inx, iny, p = sel[ok], pos[ok], inx[ok], iny[ok], p[ok]
            if len(sel) == 0:
                continue
            a = p[:, 0] - inx.astype(np.float32)
            b = p[:, 1] - iny.astype(np.float32)
            w = _weights(a, b)
            Jw = _interp(_gather(J, iny, inx, nxt.win[0], nxt.win[1], (ww, wh), cn), w, cn, W_BITS - 5, (ww, wh))
            ad = np.abs(Jw - Iw[pos]).astype(np.float32).reshape(len(sel), -1)
            ev = np.zeros(len(sel), np.float32)
            for t in range(ad.shape[1]):
                ev += ad[:, t]
            err[sel] = ev / f32(32 * ww * cn * wh)
            written[sel] = True
    return out, status, err, written
