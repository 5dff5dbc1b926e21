"""numpy statement of cudalegacy's block-matching optical flow, as libb200flow's bm.cu computes it.

fastbm(I0, I1, search_window, block_window)
    cv::cuda::FastOpticalFlowBM (modules/cudalegacy/src/bm_fast.cpp:62-88, src/cuda/bm_fast.cu:70-290).  Both frames are
    extended by search_window // 2 + block_window // 2 with cudev's reflect-101 rule (``cudev_reflect101``: one fold and
    a modulo, which differs from the CPU's iterative borderInterpolate once the border exceeds the frame).  Each pixel
    takes the candidate k = y * search_window + x whose block SAD is least, ties going to the least
    (tie_pref(k mod 128), k div 128): the reference's 128 threads each keep their first strict minimum over
    k = t, t + 128, ..., and its key-value reduceKeyVal<128> is a halving tree over lanes (16, 8, 4, 2, 1) inside each
    warp and then over warps (2, 1), each merge keeping the lower position on ties.  So among tied threads the one whose
    thread-index bits 5, 6, 0, 1, 2, 3, 4 are least, in that order of significance, wins.  Flow = (x - sr, y - sr).

calc_bm(prev, curr, block, shift, max_range, use_previous, velx, vely)
    cv::cuda::calcOpticalFlowBM (src/bm.cpp:60-202, src/cuda/bm.cu:56-160): the per-cell sequential rule over the
    spiral scan table, vectorised over cells, in int32 arithmetic where the GPU wraps.  ``counters`` (a dict) receives
    how many cells ended in each branch.
"""
from __future__ import annotations

import numpy as np

INT_MAX = 2**31 - 1
FBM_MAX_SEARCH = 109  # 4 sw^2 + 1024 bytes of shared memory must fit 48 KB in the reference's launch
FBM_MAX_BLOCK = 31    # the engine's warp keeps 32 - (block_window - 1) output columns


def cudev_reflect101(i, n: int):
    """cudev BrdReflect101 index: idx_low(idx_high(i, n), n)."""
    i = np.asarray(i, np.int64)
    last = n - 1
    hi = np.abs(last - np.abs(last - i)) % n
    return np.abs(hi) % n


def pad_cudev(img: np.ndarray, border: int) -> np.ndarray:
    r, c = img.shape
    ri = cudev_reflect101(np.arange(-border, r + border), r)
    ci = cudev_reflect101(np.arange(-border, c + border), c)
    return img[np.ix_(ri, ci)]


def tie_pref(t):
    """Rank of reference thread t (0..127) among tied threads after reduceKeyVal<128>: the warp index bit-reversed, then
    the lane bit-reversed."""
    t = np.asarray(t)
    lane = sum(((t >> b) & 1) << (4 - b) for b in range(5))
    return lane | (((t >> 5) & 1) << 6) | (((t >> 6) & 1) << 5)


def rank(k, sw: int):
    """Position of candidate k in the reference's tie order (tie_pref(k mod 128), k div 128)."""
    nq = -(-sw * sw // 128)
    k = np.asarray(k)
    return tie_pref(k % 128) * nq + k // 128


def key_layout(sw: int, bw: int):
    """(rank bits, wide): the engine packs (SAD, rank) into an int32 unless that could overflow."""
    rmax = int(rank(np.arange(sw * sw), sw).max())
    bits = rmax.bit_length()
    return bits, ((255 * bw * bw) << bits) + rmax > INT_MAX


def check_fastbm_args(sw: int, bw: int) -> bool:
    return 1 <= sw <= FBM_MAX_SEARCH and 1 <= bw <= FBM_MAX_BLOCK and bw % 2 == 1


def _box(d: np.ndarray, bw: int) -> np.ndarray:
    s = np.cumsum(np.cumsum(d, axis=0, dtype=np.int64), axis=1)
    s = np.pad(s, ((1, 0), (1, 0)))
    return s[bw:, bw:] - s[:-bw, bw:] - s[bw:, :-bw] + s[:-bw, :-bw]


def fastbm_sad(I0: np.ndarray, I1: np.ndarray, sw: int, bw: int):
    """Yield (k, D_k) with D_k the int64 block-SAD plane of candidate k (closed form)."""
    sr, br = sw // 2, bw // 2
    b = sr + br
    r, c = I0.shape
    E0 = pad_cudev(I0, b).astype(np.int32)
    E1 = pad_cudev(I1, b).astype(np.int32)
    A = E0[b - br:b + r + br, b - br:b + c + br]
    for k in range(sw * sw):
        y, x = divmod(k, sw)
        oy, ox = b - br + y - sr, b - br + x - sr
        B = E1[oy:oy + r + 2 * br, ox:ox + c + 2 * br]
        yield k, _box(np.abs(A - B), bw)


def fastbm(I0: np.ndarray, I1: np.ndarray, search_window: int = 21, block_window: int = 7) -> np.ndarray:
    """(H, W, 2) float32 flow."""
    assert I0.dtype == np.uint8 and I1.dtype == np.uint8 and I0.shape == I1.shape
    sw, bw = search_window, block_window
    assert check_fastbm_args(sw, bw)
    nr = 128 * -(-sw * sw // 128)
    best = np.full(I0.shape, np.iinfo(np.int64).max, np.int64)
    for k, D in fastbm_sad(I0, I1, sw, bw):
        np.minimum(best, D * nr + int(rank(k, sw)), out=best)
    r = best % nr
    nq = nr // 128
    k = tie_pref(r // nq) + 128 * (r % nq)  # tie_pref is its own inverse
    sr = sw // 2
    return np.stack([(k % sw - sr), (k // sw - sr)], axis=-1).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- grid BM
def spiral(W: int, H: int) -> np.ndarray:
    """The reference's scan table: (2W+1)(2H+1) - 1 offsets (x, y), origin excluded."""
    out = []
    m = min(W, H)
    for r in range(1, m + 1):  # ring of radius r, clockwise from the cell right of its top-left corner
        out += [(x, -r) for x in range(-r + 1, r + 1)]
        out += [(r, y) for y in range(-r + 1, r + 1)]
        out += [(x, r) for x in range(r - 1, -r - 1, -1)]
        out += [(-r, y) for y in range(r - 1, -r - 1, -1)]
    if W < H:  # the rest: pairs of whole rows, upper then lower
        for i in range(m, H):
            out += [(x, -(i + 1)) for x in range(-W, W + 1)]
            out += [(x, i + 1) for x in range(-W, W + 1)]
    elif W > H:  # pairs of whole columns, left then right
        for i in range(m, W):
            out += [(-(i + 1), y) for y in range(-H, H + 1)]
            out += [(i + 1, y) for y in range(-H, H + 1)]
    return np.array(out, np.int64).reshape(-1, 2)


def float2int_rn(v) -> np.ndarray:
    """__float2int_rn (cvt.rni.s32.f32): round half to even, saturating, NaN -> 0."""
    v = np.asarray(v, np.float32).astype(np.float64)
    r = np.rint(np.nan_to_num(v, nan=0.0, posinf=np.inf, neginf=-np.inf))
    return np.clip(r, -2.0**31, 2.0**31 - 1).astype(np.int64)


def wrap32(v):
    return ((np.asarray(v, np.int64) + 2**31) % 2**32) - 2**31


def vel_size(rows: int, cols: int, block, shift):
    """velSize with C division (truncation toward zero)."""
    def cdiv(a, b):
        return int(a / b) if a >= 0 else -((-a) // b)
    return cdiv(rows - block[1] + shift[1], shift[1]), cdiv(cols - block[0] + shift[0], shift[0])


def _sad(prev, curr, X1, Y1, X2, Y2, bw, bh):
    """|curr(Y1.., X1..) - prev(Y2.., X2..)| summed over the block, per cell, grouped by offset."""
    out = np.zeros(X1.shape, np.int64)
    if X1.size == 0:
        return out
    ox, oy = X2 - X1, Y2 - Y1
    pairs, inv = np.unique(np.stack([ox, oy], 1), axis=0, return_inverse=True)
    inv = inv.ravel()
    c32, p32 = curr.astype(np.int32), prev.astype(np.int32)
    ys, xs = np.arange(bh), np.arange(bw)
    for g, (dx, dy) in enumerate(pairs):
        sel = np.nonzero(inv == g)[0]
        x1, y1 = X1[sel], Y1[sel]
        if sel.size * bw * bh <= 1 << 21:
            a = c32[(y1[:, None, None] + ys[None, :, None]), (x1[:, None, None] + xs[None, None, :])]
            b = p32[(y1[:, None, None] + dy + ys[None, :, None]), (x1[:, None, None] + dx + xs[None, None, :])]
            out[sel] = np.abs(a - b).reshape(sel.size, -1).sum(1)
        else:  # an integral image of |curr - shifted prev| over the cells' bounding box
            y0, y1m, x0, x1m = y1.min(), y1.max() + bh, x1.min(), x1.max() + bw
            d = np.abs(c32[y0:y1m, x0:x1m] - p32[y0 + dy:y1m + dy, x0 + dx:x1m + dx])
            s = np.pad(np.cumsum(np.cumsum(d, 0, dtype=np.int64), 1), ((1, 0), (1, 0)))
            ry, rx = y1 - y0, x1 - x0
            out[sel] = s[ry + bh, rx + bw] - s[ry, rx + bw] - s[ry + bh, rx] + s[ry, rx]
    return out


BRANCHES = ("accepted_at_start", "accepted_in_search", "best_of_scan", "tie_averaged", "escaped",
            "escaped_after_accept")


def calc_bm(prev: np.ndarray, curr: np.ndarray, block, shift, max_range, use_previous: bool,
            velx: np.ndarray | None = None, vely: np.ndarray | None = None, counters: dict | None = None):
    """-> (velx, vely) float32 of velSize.  block / shift / max_range are (width, height)."""
    assert prev.dtype == np.uint8 and curr.dtype == np.uint8 and prev.shape == curr.shape
    bw, bh = block
    W, H = max_range
    rows, cols = prev.shape
    vr, vc = vel_size(rows, cols, block, shift)
    assert vr > 0 and vc > 0
    maxX, maxY = cols - bw, rows - bh
    accept, escape = 2 * bw * bh, 128 * bw * bh
    ii, jj = np.meshgrid(np.arange(vr), np.arange(vc), indexing="ij")
    X1, Y1 = (jj * shift[0]).ravel(), (ii * shift[1]).ravel()
    n = X1.size
    if use_previous:
        offX, offY = float2int_rn(velx).ravel(), float2int_rn(vely).ravel()
    else:
        offX = offY = np.zeros(n, np.int64)

    def in_range(X2, Y2):
        return (0 <= X2) & (X2 <= maxX) & (0 <= Y2) & (Y2 <= maxY)

    X2, Y2 = wrap32(X1 + offX), wrap32(Y1 + offY)
    dist = np.full(n, INT_MAX, np.int64)
    ok = in_range(X2, Y2)
    dist[ok] = _sad(prev, curr, X1[ok], Y1[ok], X2[ok], Y2[ok], bw, bh)
    sumx, sumy, count = offX.copy(), offY.copy(), np.ones(n, np.int64)
    search = dist > accept
    done = ~search
    accepted = np.zeros(n, bool)
    for sx, sy in spiral(W, H):
        act = ~done
        if not act.any():
            break
        dx, dy = wrap32(offX + sx), wrap32(offY + sy)
        X2, Y2 = wrap32(X1 + dx), wrap32(Y1 + dy)
        inr = act & in_range(X2, Y2)
        idx = np.nonzero(inr)[0]
        tmp = np.full(n, INT_MAX, np.int64)
        tmp[idx] = _sad(prev, curr, X1[idx], Y1[idx], X2[idx], Y2[idx], bw, bh)
        acc = inr & (tmp < accept)
        sumx[acc], sumy[acc], count[acc] = dx[acc], dy[acc], 1
        accepted |= acc
        done |= acc
        rest = inr & ~acc
        lt = rest & (tmp < dist)
        eq = rest & (tmp == dist)
        dist[lt], sumx[lt], sumy[lt], count[lt] = tmp[lt], dx[lt], dy[lt], 1
        sumx[eq], sumy[eq], count[eq] = wrap32(sumx[eq] + dx[eq]), wrap32(sumy[eq] + dy[eq]), count[eq] + 1
    esc = search & (dist > escape)
    sumx[esc], sumy[esc], count[esc] = offX[esc], offY[esc], 1
    if counters is not None:
        counters["accepted_at_start"] = int((~search).sum())
        counters["accepted_in_search"] = int((accepted & ~esc).sum())
        counters["best_of_scan"] = int((search & ~accepted & ~esc & (count == 1)).sum())
        counters["tie_averaged"] = int((search & ~accepted & ~esc & (count > 1)).sum())
        counters["escaped"] = int((esc & ~accepted).sum())
        counters["escaped_after_accept"] = int((esc & accepted).sum())
    cnt = count.astype(np.float32)
    vx = (sumx.astype(np.int32).astype(np.float32) / cnt).astype(np.float32).reshape(vr, vc)
    vy = (sumy.astype(np.int32).astype(np.float32) / cnt).astype(np.float32).reshape(vr, vc)
    return vx, vy
