"""numpy model of ``cv::cuda::interpolateFrames`` (modules/cudalegacy/src/interpolate_frames.cpp:54-111,
src/cuda/NPP_staging.cu:1648-1790 nppiStInterpolateFrames / BlendFramesKernel, :1838-1905
ForwardWarpKernel_PSF2x2, :1956-1996 NormalizeKernel / MemsetKernel, :2022-2063 nppiStVectorWarp_PSF2x2).

TEST INFRASTRUCTURE (see oracle/__init__.py).  **Parity unpinned**: the reference has no CPU
implementation and its only test (cudalegacy test_nvidia / NCV) needs opencv_extra data.  The model
reproduces the reference's defects when ``corrected=False``:
  * the 4th pass writes bwdU again (NPP_staging.cu:1779-1787), bwdV stays zero;
  * the "visible in both frames" branch samples frame0 twice (:1666);
  * MemsetKernel clears ``i*w + j`` (:1985-1996), i.e. only the first w*h floats of a pitched plane.

It is built from three stages, each rounding every float32 operation once, as ``csrc/frames.cu`` does
(it is compiled without FMA contraction):
  * ``splat``: the contributions ``value * weight`` of ForwardWarpKernel_PSF2x2 to the six accumulators
    (cov0, cov1, fwdU, fwdV, bwdU, bwdV), tap by tap and in raster order within a tap;
  * ``normalise``: the accumulators divided by their coverage, left in ``buf`` the way the engine leaves them;
  * ``blend``: the output frame from what ``buf`` holds after the call and the two frames.

``interpolate_frames(order="reference")`` follows the reference call by call (four splat passes with
their coverage clears, the bv splat accumulated onto the normalised bwdU, the coverage past w*h
accumulated a second time).  ``order="engine"`` follows ``frames.cu``: one splat into six
accumulators, then ``normalise(normalise(bwdU, c1) + bv_sum, c1b)`` and ``c + c`` for the coverage past
w*h.  Both accumulate in the order above; the GPU's float atomics add in an arbitrary order.  So:
  * the blend is exact: it is a deterministic function of ``buf`` after the call (``blend``);
  * where every contribution to an accumulator lies on the 2^-k lattice and their magnitudes sum to less
    than 2^(24-k), every partial sum is exact in float32 and every order gives the same bits
    (``terms`` / ``order_free``); then the whole call is exact;
  * otherwise an accumulator is within ``error_bound`` of the exact sum, and ``normalised_intervals``
    carries that bound through the normalisation.

Hardware rules the model states: the atomics (RED.ADD.F32.FTZ) flush subnormal contributions to zero;
the float-to-int conversion of the splat coordinate follows PTX ``cvt.rzi.s32.f32`` (NaN -> 0,
out-of-range values saturate, so an infinite coordinate drops all four taps and a NaN one lands at
column or row 0).  Not modelled: an atomic whose running sum falls into the subnormal range (it needs
cancellation below 2^-126).  The tests keep non-finite flows out of the bit-exact comparisons: a NaN
reaching the output has no defined payload.  The hardware bilinear filter is modelled with 8-bit
fractional weights, as ``frames.cu`` computes it.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

F = np.float32
PLANES = ("cov0", "cov1", "fwdU", "fwdV", "bwdU", "bwdV")
U32 = 2.0 ** -24      # unit roundoff of float32
U64 = 2.0 ** -53
NO_LATTICE = -(2 ** 20)  # ``Terms.k`` of a target without nonzero contributions
_TINY = F(2.0 ** -126)


class Contributions(NamedTuple):
    """What one accumulator receives: flat target indices into a pitched (h*s) plane and float32 values, in
    the model's accumulation order."""
    idx: np.ndarray
    val: np.ndarray


class Terms(NamedTuple):
    """Per target of one accumulator (flat, length h*s): the number of contributions, the float64 sums of the
    values and of their magnitudes, and the least k such that every contribution is a multiple of 2^-k."""
    count: np.ndarray
    exact: np.ndarray
    abs_sum: np.ndarray
    k: np.ndarray


def _ftz(x):
    return np.where(np.abs(x) < _TINY, F(0), x).astype(F)


def _f2i(p):
    """cvt.rzi.s32.f32 of an integral float: NaN -> 0, saturating at the int32 range."""
    p = np.where(np.isnan(p), 0.0, p.astype(np.float64))
    return np.clip(p, -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)


def _taps(u, v, time_scale, w, h, s):
    """The four taps of ForwardWarpKernel_PSF2x2 in frames.cu's order: (flat target, weight, in-frame mask)."""
    jj, ii = np.meshgrid(np.arange(w), np.arange(h))
    cx = (u * F(time_scale) + jj.astype(F) + F(1)).astype(F)
    cy = (v * F(time_scale) + ii.astype(F) + F(1)).astype(F)
    with np.errstate(invalid="ignore"):
        px, py = np.trunc(cx), np.trunc(cy)  # modff: integral part truncates toward zero
        dx = np.where(np.isinf(cx), F(0), cx - px).astype(F)
        dy = np.where(np.isinf(cy), F(0), cy - py).astype(F)
    tx0, ty0 = _f2i(px), _f2i(py)
    one = F(1)
    out = []
    for tx, ty, wgt in ((tx0, ty0, dx * dy), (tx0 - 1, ty0, (one - dx) * dy),
                        (tx0 - 1, ty0 - 1, (one - dx) * (one - dy)), (tx0, ty0 - 1, dx * (one - dy))):
        ok = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
        out.append(((ty * s + tx)[ok], wgt.astype(F)[ok], ok))
    return out


def splat(fu, fv, bu, bv, pos, w, h, s):
    """The contributions of the forward splat (fu, fv at time pos) and the backward splat (bu, bv at 1 - pos)
    to the six accumulators, as a dict plane name -> Contributions (value * weight rounded, then flushed)."""
    pos = F(pos)
    res = {}
    for cov, (nu, nv), (a, b), ts in (("cov0", ("fwdU", "fwdV"), (fu, fv), pos),
                                      ("cov1", ("bwdU", "bwdV"), (bu, bv), F(1) - pos)):
        a, b = np.asarray(a, F), np.asarray(b, F)
        taps = _taps(a, b, ts, w, h, s)
        idx = np.concatenate([t[0] for t in taps])
        res[cov] = Contributions(idx, _ftz(np.concatenate([t[1] for t in taps])))
        res[nu] = Contributions(idx, _ftz(np.concatenate([(a[t[2]] * t[1]).astype(F) for t in taps])))
        res[nv] = Contributions(idx, _ftz(np.concatenate([(b[t[2]] * t[1]).astype(F) for t in taps])))
    return res


def accumulate(c: Contributions, n, dst=None):
    """float32 sum of the contributions onto ``dst`` (zeros of length n), one rounding per addition in the
    given order, like a serialised stream of atomics."""
    dst = np.zeros(n, F) if dst is None else dst
    np.add.at(dst, c.idx, c.val)  # unbuffered: element by element in the array dtype
    return dst


def _lattice_k(val):
    """Least k with val a multiple of 2^-k, per float32 value; NO_LATTICE for zeros."""
    bits = np.ascontiguousarray(val, F).view(np.int32)
    E = (bits >> 23) & 0xFF
    M = (bits & 0x7FFFFF) | ((E > 0).astype(np.int32) << 23)  # |val| = M * 2^(max(E, 1) - 150)
    tz = np.bitwise_count((M & -M) - 1).astype(np.int32)  # trailing zeros of M
    return np.where(M > 0, 150 - np.maximum(E, 1) - tz, NO_LATTICE).astype(np.int64)


def terms(c: Contributions, n) -> Terms:
    """Contribution data of one accumulator per target (flat, length n)."""
    v = c.val.astype(np.float64)
    count = np.bincount(c.idx, minlength=n)
    exact = np.bincount(c.idx, weights=v, minlength=n)
    abs_sum = np.bincount(c.idx, weights=np.abs(v), minlength=n)
    k = np.full(n, NO_LATTICE, np.int64)
    np.maximum.at(k, c.idx, _lattice_k(c.val))
    return Terms(count, exact, abs_sum, k)


def order_free(t: Terms):
    """True where every partial sum of every order is exact in float32: all contributions are multiples of
    2^-k and the magnitudes sum to less than 2^(24-k), so each partial sum is an integer below 2^24 times
    2^-k.  Then the float64 sum ``t.exact`` is exact too."""
    return t.abs_sum < np.ldexp(1.0, np.minimum(24 - t.k, 1000).astype(np.int64))


def _gamma(m, u):
    m = np.maximum(m, 0).astype(np.float64)
    return m * u / (1.0 - m * u)


def error_bound(t: Terms):
    """Bound on |fl32 sum in any order - t.exact|: gamma_{n-1} sum|a_i| (recursive summation from 0 in any
    order) plus the float64 sum's own gamma_{n-1} sum|a_i|, with slack for the float64 evaluation."""
    return (_gamma(t.count - 1, U32) + _gamma(t.count - 1, U64)) * t.abs_sum * (1.0 + 2.0 ** -40)


def normalise(acc, corrected, w, h, s):
    """frames.cu's normalisation of the six raw accumulators (flat, (6, h*s)): returns buf (6, h*s) as the
    engine leaves it.  Reference mode: ``c + c`` for the coverage past w*h (accumulated twice by the
    reference), ``normalise(normalise(bwdU, c1) + bwdV, c1b)`` for the 4th pass, bwdV zero."""
    buf = np.array(acc, F).reshape(6, h, s)
    c0, c1, fu, fv, bu, bv = (p[:, :w] for p in buf)
    inv = lambda c: np.where(c == 0, F(1), F(1) / np.where(c == 0, F(1), c)).astype(F)
    if corrected:
        i0, i1 = inv(c0), inv(c1)
        u, v, ur, vr = fu * i0, fv * i0, bu * i1, bv * i1
        c0b, c1b = c0, c1
    else:
        cleared = _cleared(w, h, s)
        c0b = np.where(cleared, c0, c0 + c0).astype(F)
        c1b = np.where(cleared, c1, c1 + c1).astype(F)
        u, v = fu * inv(c0), fv * inv(c0b)
        ur = ((bu * inv(c1)).astype(F) + bv).astype(F) * inv(c1b)
        vr = np.zeros_like(bv)
    for k, p in enumerate((c0b, c1b, u, v, ur, vr)):
        buf[k, :, :w] = p
    return buf.reshape(6, h * s)


def _cleared(w, h, s):
    """The pixels MemsetKernel clears: flat offset i*s + j below w*h."""
    jj, ii = np.meshgrid(np.arange(w), np.arange(h))
    return ii * s + jj < w * h


def _tex_linear(img, y, x):
    h, w = img.shape
    xb, yb = (x - F(0.5)).astype(F), (y - F(0.5)).astype(F)
    fx, fy = np.floor(xb), np.floor(yb)
    ax = (np.floor((xb - fx) * F(256) + F(0.5)) * F(1 / 256)).astype(F)
    ay = (np.floor((yb - fy) * F(256) + F(0.5)) * F(1 / 256)).astype(F)
    x0 = np.clip(fx, -2, w + 1).astype(np.int64)
    y0 = np.clip(fy, -2, h + 1).astype(np.int64)
    xa, xc = np.clip(x0, 0, w - 1), np.clip(x0 + 1, 0, w - 1)
    ya, yc = np.clip(y0, 0, h - 1), np.clip(y0 + 1, 0, h - 1)
    one = F(1)
    return ((one - ax) * (one - ay) * img[ya, xa] + ax * (one - ay) * img[ya, xc] + (one - ax) * ay * img[yc, xa] +
            ax * ay * img[yc, xc]).astype(F)


def blend_branches(cov0, cov1):
    """(both, first only, second only) masks of BlendFramesKernel from the coverages left in buf."""
    b0, b1 = cov0 > F(1e-4), cov1 > F(1e-4)
    return b0 & b1, b0 & ~b1, ~b0


def blend(frame0, frame1, planes, pos, corrected=False):
    """BlendFramesKernel from the six (h, w) planes of buf after the call (cov0, cov1, u, v, ur, vr)."""
    frame0, frame1 = np.asarray(frame0, F), np.asarray(frame1, F)
    h, w = frame0.shape
    o0, o1, u, v, ur, vr = (np.asarray(p, F) for p in planes)
    pos = F(pos)
    jj, ii = np.meshgrid(np.arange(w), np.arange(h))
    x, y = jj.astype(F) + F(0.5), ii.astype(F) + F(0.5)
    one = F(1)
    both_m, first_m, _ = blend_branches(o0, o1)
    with np.errstate(invalid="ignore", over="ignore"):
        a = _tex_linear(frame0, y - v * pos, x - u * pos)
        second = frame1 if corrected else frame0
        bsample = _tex_linear(second, y + v * (one - pos), x + u * (one - pos))
        both = (a * (one - pos) + bsample * pos).astype(F)
        c = _tex_linear(frame1, y - vr * (one - pos), x - ur * (one - pos))
    return np.where(both_m, both, np.where(first_m, a, c)).astype(F)


def _vector_warp(con, cov, norm, dst, w, h, s):
    """nppiStVectorWarp_PSF2x2_32f_C1: clear (by width!), splat, normalise."""
    norm[: w * h] = 0  # MemsetKernel indexes i*w + j
    accumulate(con[cov], norm.size, norm)
    accumulate(dst[1], norm.size, dst[0])
    inv = np.where(norm == 0, F(1), (F(1) / np.where(norm == 0, F(1), norm))).astype(F)
    # NormalizeKernel touches columns < w only
    d2, i2 = dst[0].reshape(h, s), inv.reshape(h, s)
    d2[:, :w] = (d2[:, :w] * i2[:, :w]).astype(F)


def interpolate_frames(frame0, frame1, fu, fv, bu, bv, pos, stride=None, corrected=False, order="reference"):
    """Returns (new_frame (h, w), buf (6, h, stride)) with buf = cov0, cov1, fwdU, fwdV, bwdU, bwdV.
    ``order``: "reference" (the reference's passes) or "engine" (frames.cu's); see the module docstring."""
    h, w = np.shape(frame0)
    s = w if stride is None else int(stride)
    frame0, frame1, fu, fv, bu, bv = (np.ascontiguousarray(a, F) for a in (frame0, frame1, fu, fv, bu, bv))
    con = splat(fu, fv, bu, bv, pos, w, h, s)
    if order == "engine":
        buf = normalise([accumulate(con[p], h * s) for p in PLANES], corrected, w, h, s)
    elif order == "reference":
        buf = np.zeros((6, h * s), F)  # buf.setTo(0)
        cov0, cov1, fwdU, fwdV, bwdU, bwdV = buf
        if corrected:
            for p, dst in zip(PLANES, buf):
                accumulate(con[p], h * s, dst)
            for dst, cov in ((fwdU, cov0), (fwdV, cov0), (bwdU, cov1), (bwdV, cov1)):
                inv = np.where(cov == 0, F(1), F(1) / np.where(cov == 0, F(1), cov)).astype(F)
                dst *= inv
        else:
            _vector_warp(con, "cov0", cov0, (fwdU, con["fwdU"]), w, h, s)
            _vector_warp(con, "cov0", cov0, (fwdV, con["fwdV"]), w, h, s)
            _vector_warp(con, "cov1", cov1, (bwdU, con["bwdU"]), w, h, s)
            _vector_warp(con, "cov1", cov1, (bwdU, con["bwdV"]), w, h, s)  # sic: bwdU again
    else:
        raise ValueError(order)
    B = buf.reshape(6, h, s)
    out = blend(frame0, frame1, B[:, :, :w], pos, corrected)
    return out, B


# ------------------------------------------------------------------------------------- interval bounds
_SLACK = 2.0 ** -45  # covers the float64 evaluation of the bounds themselves


def _round(lo, hi, mag):
    """Float32 values every fl32(x) can take for a real x in [lo, hi]; lo and hi were computed in float64 from
    terms of magnitude up to ``mag``, so they are first widened by the float64 error."""
    with np.errstate(over="ignore", invalid="ignore"):
        lo = (lo - mag * _SLACK).astype(F).astype(np.float64)
        hi = (hi + mag * _SLACK).astype(F).astype(np.float64)
    return lo, hi


def _recip(cl, ch):
    """fl(1/c) for c in [cl, ch], and ``scale == 0 -> 1``: NaN where the interval straddles 0 with c not
    known to be exactly 0."""
    zero = (cl == 0) & (ch == 0)
    det = (cl > 0) | (ch < 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        a, b = 1.0 / ch, 1.0 / cl
        lo, hi = _round(np.minimum(a, b), np.maximum(a, b), np.maximum(np.abs(a), np.abs(b)))
    lo = np.where(zero, 1.0, np.where(det, lo, np.nan))
    hi = np.where(zero, 1.0, np.where(det, hi, np.nan))
    return lo, hi


def _mul(a, b):
    """fl(x * y) for x in a = (lo, hi), y in b = (lo, hi)."""
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.stack([a[0] * b[0], a[0] * b[1], a[1] * b[0], a[1] * b[1]])
        return _round(p.min(0), p.max(0), np.abs(p).max(0))


def _add(a, b):
    with np.errstate(invalid="ignore", over="ignore"):
        return _round(a[0] + b[0], a[1] + b[1], np.maximum(np.abs(a[0]), np.abs(a[1])) +
                      np.maximum(np.abs(b[0]), np.abs(b[1])))


def normalised_intervals(T, corrected, w, h, s):
    """Bounds on the six (h, w) planes the engine leaves in buf, whatever the order of its atomics.

    ``T``: dict plane -> Terms of the engine's accumulators.  Returns a list of six (lo, hi) float64 pairs;
    both are NaN where a coverage interval contains 0 and the result is therefore not determined."""
    def acc(p):
        t = T[p]
        B = error_bound(t)
        lo, hi = t.exact - B, t.exact + B
        with np.errstate(invalid="ignore"):
            lo = lo - (np.abs(t.exact) + B) * _SLACK
            hi = hi + (np.abs(t.exact) + B) * _SLACK
        return lo.reshape(h, s)[:, :w], hi.reshape(h, s)[:, :w]

    c0, c1 = acc("cov0"), acc("cov1")
    fu, fv, bu, bv = acc("fwdU"), acc("fwdV"), acc("bwdU"), acc("bwdV")
    if corrected:
        i0, i1 = _recip(*c0), _recip(*c1)
        return [c0, c1, _mul(fu, i0), _mul(fv, i0), _mul(bu, i1), _mul(bv, i1)]
    cleared = _cleared(w, h, s)
    twice = lambda c: (np.where(cleared, c[0], 2 * c[0]), np.where(cleared, c[1], 2 * c[1]))  # c + c is exact
    c0b, c1b = twice(c0), twice(c1)
    ur = _mul(_add(_mul(bu, _recip(*c1)), bv), _recip(*c1b))
    z = np.zeros((h, w))
    return [c0b, c1b, _mul(fu, _recip(*c0)), _mul(fv, _recip(*c0b)), ur, (z, z)]
