"""numpy model of the reference's Brox et al. optical flow, ``cv::cuda::BroxOpticalFlow``
(modules/cudaoptflow/src/brox.cpp -> modules/cudalegacy/src/cuda/NCVBroxOpticalFlow.cu +
NPP_staging.cu filters / resizers).

TEST INFRASTRUCTURE (see oracle/__init__.py).  **Parity unpinned**: the reference has no CPU
implementation of Brox, its golden vector (opencv_extra opticalflow/brox_optical_flow_cc20.bin) is
not in the container and the CUDA reference cannot be built here; this restatement is checked only
for self-consistency (recovers synthetic ground truth, no NaNs) and the CUDA engine is checked
against it.  One documented deviation: the reference samples images through hardware bilinear
texture filtering (9-bit fixed-point weights); the model (and the engine) use exact float32 weights.

Every rounding is the engine's (opencv_contrib_b200/csrc/brox.cu): ``fmaf`` exactly where the kernels fuse a multiply
and an add, one rounding per operation elsewhere.  The one operation CUDA does not specify bit for bit is the data
term's ``rsqrtf`` (MUFU.RSQ, up to 2 ulp).  ``calc(..., rsqrt="exact")`` rounds it correctly, as the engine does with
aux_path 1, and must equal the engine bit for bit.  ``rsqrt="perturbed"`` moves the correctly rounded value by -2..+2
ulp in a fixed pattern hashed from the level, the inner step and the pixel: how far the flow moves under that is the
yardstick for the production path (aux_path 0).  The C restatement oracle/brox_model.c (loaded by
oracle/brox_model_native.py) does the same operations and is what runs at full size; this file is the readable
statement and checks it at small sizes.

``calc(..., counters=dict)`` fills ``COUNTER_NAMES``: ``mirrored`` = warped fetches (per pixel and level) whose bilinear
cell needed mirror addressing, ``degenerate`` = supersampled pixels with an empty source span on an axis
(iXEnd == iXBegin), ``levels`` = levels solved.

Citations: NB = opencv_contrib/modules/cudalegacy/src/cuda/NCVBroxOpticalFlow.cu,
           NS = opencv_contrib/modules/cudalegacy/src/cuda/NPP_staging.cu.
"""
from __future__ import annotations

import math

import numpy as np

from .denselk_model import fmaf

F = np.float32
EPS2 = F(1e-6)  # NB:78
OMEGA = F(1.99)  # NB:914
COUNTER_NAMES = ("mirrored", "degenerate", "levels")
RSQRT_MODES = ("exact", "perturbed")


class BroxParams:
    """Defaults of cv::cuda::BroxOpticalFlow::create (cudaoptflow.hpp:179-185)."""

    def __init__(self, alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=5, outer_iterations=150,
                 solver_iterations=10):
        self.alpha, self.gamma, self.scale_factor = alpha, gamma, scale_factor
        self.inner_iterations, self.outer_iterations, self.solver_iterations = (
            inner_iterations, outer_iterations, solver_iterations)


def pyramid_sizes(h: int, w: int, scale_factor: float, outer_iterations: int):
    """NB:730-785: ceilf(src * scale), cumulative float32 scale, stop at <= 15 px or the level cap."""
    sizes = [(h, w)]
    sf = F(scale_factor)
    scale = F(1.0) * sf
    pw, ph = w, h
    while pw > 15 and ph > 15 and len(sizes) < outer_iterations:
        lw = int(math.ceil(float(F(w) * scale)))
        lh = int(math.ceil(float(F(h) * scale)))
        sizes.append((lh, lw))
        scale = F(scale * sf)
        pw, ph = lw, lh
    return sizes


def _cmp_pow2(A, M, K):
    """Sign of A^2 * M - 2^K, exactly, for uint64 arrays A < 2^27, M < 2^25 and K >= 27 (int arrays)."""
    A, M, K = (np.asarray(v, np.uint64) for v in (A, M, K))
    A2 = A * A
    hi, lo = A2 >> np.uint64(26), A2 & np.uint64((1 << 26) - 1)
    lm = lo * M
    Q = hi * M + (lm >> np.uint64(26))
    rem = lm & np.uint64((1 << 26) - 1)
    T = np.uint64(1) << (K - np.uint64(26))
    return np.where(Q < T, -1, np.where((Q > T) | (rem > 0), 1, 0))


def rsqrt_is_correctly_rounded(x, r):
    """Exact integer check that float32 r is 1/sqrt(x) rounded to nearest, for positive finite float32 x (normal or
    subnormal) and normal r: the exact value lies strictly between the midpoints of r and its neighbours, i.e.
    m_lo^2 * x < 1 < m_hi^2 * x with every product taken in integers."""
    x, r = np.asarray(x, F), np.asarray(r, F)
    xb, rb = x.view(np.int32).astype(np.int64), r.view(np.int32).astype(np.int64)
    xe, re_ = xb >> 23, rb >> 23
    M = np.where(xe == 0, xb & 0x7FFFFF, (xb & 0x7FFFFF) | 0x800000)      # x = M * 2^Ex
    Ex = np.where(xe == 0, -149, xe - 150)
    R = (rb & 0x7FFFFF) | 0x800000                                       # r = R * 2^Er, 2^23 <= R < 2^24
    Er = re_ - 150
    # m_hi = (2R + 1) * 2^(Er - 1); m_lo = (2R - 1) * 2^(Er - 1), or (4R - 1) * 2^(Er - 2) when r is a power of two
    pow2 = R == 0x800000
    A_lo = np.where(pow2, 4 * R - 1, 2 * R - 1)
    S_lo = np.where(pow2, Er - 2, Er - 1)
    # m^2 * x < 1  <=>  A^2 * M < 2^-(2S + Ex)
    lo_ok = _cmp_pow2(A_lo, M, -(2 * S_lo + Ex)) < 0
    hi_ok = _cmp_pow2(2 * R + 1, M, -(2 * (Er - 1) + Ex)) > 0
    return lo_ok & hi_ok & (re_ > 0) & (re_ < 255)


def rsqrt_rn(x):
    """1/sqrt(x) correctly rounded to float32 (__frsqrt_rn) for positive float32 x.  Rounding the double result again
    can misround, so the candidate is checked exactly and moved by one ulp where it is not the nearest float."""
    x = np.asarray(x, F)
    r = (1.0 / np.sqrt(x.astype(np.float64))).astype(F)
    fin = np.isfinite(x) & (x > 0)
    if not fin.all():
        raise ValueError("rsqrt_rn: argument must be positive and finite")
    bad = ~rsqrt_is_correctly_rounded(x, r)
    for i in np.flatnonzero(bad.ravel()):
        xi = x.ravel()[i]
        for c in (np.nextafter(r.ravel()[i], F(0)), np.nextafter(r.ravel()[i], F(np.inf))):
            if rsqrt_is_correctly_rounded(xi, c):
                r.ravel()[i] = c
                break
        else:
            raise AssertionError(f"rsqrt_rn: no correctly rounded neighbour for {xi!r}")
    return r


def perturb_ulps(level: int, inner: int, n: int) -> np.ndarray:
    """The fixed -2..+2 ulp pattern of rsqrt="perturbed" for pixels 0..n-1 (row-major) of one inner step."""
    with np.errstate(over="ignore"):
        h = np.arange(n, dtype=np.uint32) * np.uint32(2654435761)
        h ^= np.uint32((level * 40503 + inner * 9973 + 1) & 0xFFFFFFFF)
        h ^= h >> np.uint32(15)
        h *= np.uint32(2246822519)
        h ^= h >> np.uint32(13)
    return (h % np.uint32(5)).astype(np.int64) - 2


def data_rsqrt(r2, rsqrt="exact", level=0, inner=0):
    r = rsqrt_rn(r2)
    if rsqrt == "exact":
        return r
    if rsqrt != "perturbed":
        raise ValueError(rsqrt)
    k = perturb_ulps(level, inner, r.size).reshape(r.shape)
    normal = (r > np.finfo(F).tiny) & np.isfinite(r)
    bits = r.view(np.int32).astype(np.int64) + np.where(normal, k, 0)
    return bits.astype(np.int32).view(F)


def resize_supersample(src: np.ndarray, dh: int, dw: int, scale: float, cnt=None) -> np.ndarray:
    """resizeSuperSample_32f (NS:2073-2149) with scaleX = scaleY = 1/factor, k_brox_supersample's roundings."""
    sh, sw = src.shape
    s = F(scale)
    out = np.zeros((dh, dw), F)

    def ranges(n_dst, n_src):
        i = np.arange(n_dst, dtype=F)
        b = np.maximum(fmaf(i, s, -s), F(0)).astype(F)
        e = np.minimum(fmaf(i, s, s), F(n_src) - F(1)).astype(F)
        fb = np.floor(b).astype(F)
        ce = np.ceil(e).astype(F)
        return b, e, fb, ce, fb.astype(np.int64), ce.astype(np.int64)

    xb, xe, fxb, cxe, ixb, ixe = ranges(dw, sw)
    yb, ye, fyb, cye, iyb, iye = ranges(dh, sh)
    if cnt is not None:
        cnt["degenerate"] += int(((ixe == ixb)[None, :] | (iye == iyb)[:, None]).sum())
    w0x = ((F(1.0) - xb) + fxb).astype(F)
    w1x = (cxe - xe).astype(F)

    def line(row):
        # ss_line for every dst x of src row `row`; iXEnd == iXBegin runs no inner tap but still adds the last one
        # at ixb + 1, like iXEnd == iXBegin + 1
        wsum = w0x
        acc = (row[ixb] * w0x).astype(F)
        last_at = np.maximum(ixe, ixb + 1)
        for k in range(1, int((last_at - ixb).max()) + 1):
            pos = ixb + k
            v = row[np.minimum(pos, sw - 1)]
            inner = pos < ixe
            acc = np.where(inner, acc + v, acc).astype(F)
            wsum = np.where(inner, wsum + F(1.0), wsum).astype(F)
            last = pos == last_at
            acc = np.where(last, fmaf(w1x, v, acc), acc)
            wsum = np.where(last, wsum + w1x, wsum).astype(F)
        return (acc / wsum).astype(F)

    for y in range(dh):
        w0 = F(F(F(1.0) - yb[y]) + fyb[y])
        w1 = F(cye[y] - ye[y])
        wsum = w0
        acc = (line(src[iyb[y]]) * w0).astype(F)
        yy = iyb[y] + 1
        while yy < iye[y]:
            acc = (acc + line(src[yy])).astype(F)
            wsum = F(wsum + F(1.0))
            yy += 1
        acc = fmaf(w1, line(src[min(yy, sh - 1)]), acc)
        wsum = F(wsum + w1)
        out[y] = acc / wsum
    return out


def _mirror_filter_idx(i, n):
    """getValueMirrorRow/Column (NS:1433-1447): i < 0 -> 1 - i (asymmetric!), i >= n -> 2n - i - 1."""
    i = np.where(i < 0, 1 - i, i)
    i = np.where(i >= n, 2 * n - i - 1, i)
    return np.clip(i, 0, n - 1)


def filter5(src: np.ndarray, axis: int) -> np.ndarray:
    """FilterRow/ColumnBorderMirror_32f_C1R with {1,-8,0,8,-1} * 1/12, anchor 2 (NS:1449-1501; NB:843-868).
    The products by +-1, +-8 and 0 are exact, so the kernels' contraction of the taps cannot change a bit."""
    k = np.array([1.0, -8.0, 0.0, 8.0, -1.0], F)
    n = src.shape[axis]
    idx = np.arange(n)
    acc = np.zeros_like(src)
    for m in range(5):
        j = _mirror_filter_idx(idx + m - 2, n)
        acc = acc + np.take(src, j, axis=axis) * k[m]
    return (acc * F(1.0 / 12.0)).astype(F)


def _mirror_tex(i, n):
    """cudaAddressModeMirror on texel indices: -1 -> 0, -2 -> 1, n -> n-1, n+1 -> n-2 (period 2n)."""
    i = np.mod(i, 2 * n)
    return np.where(i >= n, 2 * n - 1 - i, i)


def tex_bilinear_mirror(img: np.ndarray, xn, yn, cnt=None):
    """Normalised-coordinate, linear-filtered, mirror-addressed texture fetch (NB:829-830,870-876), with exact
    float32 weights: tex_bilinear in brox.cu.  The cell index is clamped to +-1e6 before the integer conversion."""
    h, w = img.shape
    xb = fmaf(xn, F(w), F(-0.5))
    yb = fmaf(yn, F(h), F(-0.5))
    fx0, fy0 = np.floor(xb), np.floor(yb)
    ax, ay = (xb - fx0).astype(F), (yb - fy0).astype(F)
    bx, by = (F(1) - ax).astype(F), (F(1) - ay).astype(F)
    x0 = np.clip(fx0, F(-1.0e6), F(1.0e6)).astype(np.int64)
    y0 = np.clip(fy0, F(-1.0e6), F(1.0e6)).astype(np.int64)
    if cnt is not None:
        cnt["mirrored"] += int(((x0 < 0) | (x0 + 1 >= w) | (y0 < 0) | (y0 + 1 >= h)).sum())
    xa, xc = _mirror_tex(x0, w), _mirror_tex(x0 + 1, w)
    ya, yc = _mirror_tex(y0, h), _mirror_tex(y0 + 1, h)
    top = fmaf(bx, img[ya, xa], (ax * img[ya, xc]).astype(F))
    bot = fmaf(bx, img[yc, xa], (ax * img[yc, xc]).astype(F))
    return fmaf(by, top, (ay * bot).astype(F))


def bicubic_coeff(x_):
    """brox_bicubic_coeff: Keys a = -0.5 with k_brox_prolong's fused multiply-adds."""
    x = np.abs(np.asarray(x_, F))
    near = fmaf((x * x).astype(F), fmaf(x, F(1.5), F(-2.5)), F(1.0))
    far = fmaf(x, fmaf(x, fmaf(x, F(-0.5), F(2.5)), F(-4.0)), F(2.0))
    return np.where(x <= F(1), near, np.where(x < F(2), far, F(0))).astype(F)


def resize_bicubic(src: np.ndarray, dh: int, dw: int, scale: float, mul) -> np.ndarray:
    """resizeBicubic (NS:2172-2231) times ScaleVector's factor: taps ceil(x-2)..floor(x+2) clamped to the ROI, Keys
    a=-0.5, sum / wsum, point texture with mirror addressing (never reached because of the clamp).  x = scale * ix is
    never rounded on its own (k_brox_prolong fuses it into x - 2, x + 2 and x - cx)."""
    sh, sw = src.shape
    s = F(scale)
    ys, xs = np.mgrid[0:dh, 0:dw]
    fx, fy = xs.astype(F), ys.astype(F)
    xmin = np.maximum(np.ceil(fmaf(fx, s, F(-2))), F(0))
    xmax = np.minimum(np.floor(fmaf(fx, s, F(2))), F(sw) - F(1))
    ymin = np.maximum(np.ceil(fmaf(fy, s, F(-2))), F(0))
    ymax = np.minimum(np.floor(fmaf(fy, s, F(2))), F(sh) - F(1))
    acc = np.zeros((dh, dw), F)
    wsum = np.zeros((dh, dw), F)
    for j in range(5):
        cy = (ymin + F(j)).astype(F)
        my = cy <= ymax
        wy = bicubic_coeff(fmaf(fy, s, -cy))
        cyi = np.clip(cy.astype(np.int64), 0, sh - 1)
        for i in range(5):
            cx = (xmin + F(i)).astype(F)
            m = my & (cx <= xmax)
            wgt = (bicubic_coeff(fmaf(fx, s, -cx)) * wy).astype(F)
            cxi = np.clip(cx.astype(np.int64), 0, sw - 1)
            acc = np.where(m, fmaf(wgt, src[cyi, cxi], acc), acc)
            wsum = np.where(m, wsum + wgt, wsum).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where(wsum == 0, F(0), acc / wsum).astype(F)
    return (out * F(mul)).astype(F)


def _mirror_load(a: np.ndarray, dy: int, dx: int) -> np.ndarray:
    """load_array_element (NB:238-249): neighbour (i+dx, j+dy) with mirror i<0 -> -i-1, i>=w -> 2w-i-1."""
    h, w = a.shape
    ii = np.arange(w) + dx
    jj = np.arange(h) + dy
    ii = np.maximum(ii, -ii - 1)
    ii = np.minimum(ii, w - ii + w - 1)
    jj = np.maximum(jj, -jj - 1)
    jj = np.minimum(jj, h - jj + h - 1)
    return a[np.ix_(np.clip(jj, 0, h - 1), np.clip(ii, 0, w - 1))]


def _diffusivity(u_x, v_x, u_y, v_y):
    s = fmaf(u_x, u_x, (v_x * v_x).astype(F))
    s = fmaf(u_y, u_y, s)
    s = fmaf(v_y, v_y, s)
    return (F(0.5) / np.sqrt((s + EPS2).astype(F))).astype(F)


def warp_terms(u, v, I0, I1, Ix, Ixx, Ix0, Iy, Iyy, Iy0, Ixy, cnt=None):
    """k_brox_warp_terms: the texture fetches of prepare_sor_stage_1 (NB:352-383), once per level."""
    h, w = u.shape
    jg, ig = np.mgrid[0:h, 0:w]
    x = (ig.astype(F) + F(0.5)).astype(F)
    y = (jg.astype(F) + F(0.5)).astype(F)
    wx = ((x + u) / F(w)).astype(F)
    wy = ((y + v) / F(h)).astype(F)
    xn = (x / F(w)).astype(F)
    yn = (y / F(h)).astype(F)
    ix = tex_bilinear_mirror(Ix, wx, wy, cnt)
    iy = tex_bilinear_mirror(Iy, wx, wy)
    Iz = (tex_bilinear_mirror(I1, wx, wy) - tex_bilinear_mirror(I0, xn, yn)).astype(F)
    ixz = (ix - tex_bilinear_mirror(Ix0, xn, yn)).astype(F)
    ixy = tex_bilinear_mirror(Ixy, wx, wy)
    ixx = tex_bilinear_mirror(Ixx, wx, wy)
    iyz = (iy - tex_bilinear_mirror(Iy0, xn, yn)).astype(F)
    iyy = tex_bilinear_mirror(Iyy, wx, wy)
    return Iz, ix, ixz, ixy, ixx, iy, iyz, iyy


def prepare_sor(u, v, du, dv, W, alpha, gamma, rsqrt="exact", level=0, inner=0):
    """prepare_sor_stage_1_tex + prepare_sor_stage_2 (NB:340-473): brox_prepare_chunk.  W = warp_terms(...)."""
    h, w = u.shape
    alpha, gamma = F(alpha), F(gamma)
    Iz, ix, ixz, ixy, ixx, iy, iyz, iyy = W
    q0 = fmaf(dv, iy, fmaf(du, ix, Iz))
    q1 = fmaf(dv, ixy, fmaf(du, ixx, ixz))
    q2 = fmaf(dv, iyy, fmaf(du, ixy, iyz))
    r2 = (fmaf(q0, q0, (gamma * fmaf(q1, q1, (q2 * q2).astype(F))).astype(F)) + EPS2).astype(F)
    data = (F(0.5) * data_rsqrt(r2, rsqrt, level, inner)).astype(F)
    data = (data / alpha).astype(F)

    def n(a, dy, dx):
        return _mirror_load(a, dy, dx)
    # diffusivity_along_x (NB:188-204): derivative between (i,j) and (i-1,j); left-to-right sums of tile loads
    u_x = u + du - n(u, 0, -1) - n(du, 0, -1)
    v_x = v + dv - n(v, 0, -1) - n(dv, 0, -1)
    u_y = F(0.25) * (n(u, 1, 0) + n(du, 1, 0) + n(u, 1, -1) + n(du, 1, -1) - n(u, -1, 0) - n(du, -1, 0)
                     - n(u, -1, -1) - n(du, -1, -1))
    v_y = F(0.25) * (n(v, 1, 0) + n(dv, 1, 0) + n(v, 1, -1) + n(dv, 1, -1) - n(v, -1, 0) - n(dv, -1, 0)
                     - n(v, -1, -1) - n(dv, -1, -1))
    sx = _diffusivity(u_x, v_x, u_y, v_y)
    # diffusivity_along_y (NB:216-227): derivative between (i,j) and (i,j-1)
    u_y = u + du - n(u, -1, 0) - n(du, -1, 0)
    v_y = v + dv - n(v, -1, 0) - n(dv, -1, 0)
    u_x = F(0.25) * (n(u, 0, 1) + n(u, -1, 1) + n(du, 0, 1) + n(du, -1, 1) - n(u, 0, -1) - n(u, -1, -1)
                     - n(du, 0, -1) - n(du, -1, -1))
    v_x = F(0.25) * (n(v, 0, 1) + n(v, -1, 1) + n(dv, 0, 1) + n(dv, -1, 1) - n(v, 0, -1) - n(v, -1, -1)
                     - n(dv, 0, -1) - n(dv, -1, -1))
    sy = _diffusivity(u_x, v_x, u_y, v_y)
    sx[:, 0] = 0
    sy[0, :] = 0
    num_dudv = (data * fmaf(ix, iy, ((gamma * ixy).astype(F) * (ixx + iyy)).astype(F))).astype(F)
    num_u = (data * fmaf(ix, Iz, (gamma * fmaf(ixx, ixz, (ixy * iyz).astype(F))).astype(F))).astype(F)
    num_v = (data * fmaf(iy, Iz, (gamma * fmaf(ixy, ixz, (iyy * iyz).astype(F))).astype(F))).astype(F)
    den_u = fmaf(ix, ix, (gamma * fmaf(ixy, ixy, (ixx * ixx).astype(F))).astype(F))
    den_v = fmaf(iy, iy, (gamma * fmaf(ixy, ixy, (iyy * iyy).astype(F))).astype(F))
    # stage 2: + sx(i) + sx(i+1) + sy(j) + sy(j+1), zero beyond the image
    sxr = np.zeros_like(sx)
    sxr[:, :-1] = sx[:, 1:]
    syu = np.zeros_like(sy)
    syu[:-1, :] = sy[1:, :]
    ssum = (((sx + sxr) + sy) + syu).astype(F)
    inv_u = (F(1.0) / fmaf(data, den_u, ssum)).astype(F)
    inv_v = (F(1.0) / fmaf(data, den_v, ssum)).astype(F)
    return sx, sy, inv_u, inv_v, num_dudv, num_u, num_v


def sor_pass(is_black, u, v, du, dv, sx, sy, inv_u, inv_v, num_u, num_v, num_dudv, omega=OMEGA):
    """sor_pass<isBlack> (NB:479-554) as brox_sor_cell rounds it: neighbours clamped at borders, s_right / s_up zero
    at the far edges."""
    h, w = u.shape
    jj, ii = np.mgrid[0:h, 0:w]

    def sh(a, dy, dx):
        return a[np.clip(jj + dy, 0, h - 1), np.clip(ii + dx, 0, w - 1)]

    s_l, s_d = sx, sy
    s_r = np.where(ii < w - 1, sh(sx, 0, 1), F(0)).astype(F)
    s_u = np.where(jj < h - 1, sh(sy, 1, 0), F(0)).astype(F)
    ssum = (((s_l + s_r) + s_u) + s_d).astype(F)
    omo = F(F(1.0) - omega)
    U, V = (u + du).astype(F), (v + dv).astype(F)

    def numer(A, Asum, num):
        t = (s_l * sh(A, 0, -1)).astype(F)
        t = fmaf(s_u, sh(A, 1, 0), t)
        t = fmaf(s_r, sh(A, 0, 1), t)
        t = fmaf(s_d, sh(A, -1, 0), t)
        return ((t - Asum) - num).astype(F)

    t = fmaf(-num_dudv, dv, numer(U, (u * ssum).astype(F), num_u))
    du_new = fmaf((omega * inv_u).astype(F), t, (omo * du).astype(F))
    t = fmaf(-num_dudv, du_new, numer(V, (v * ssum).astype(F), num_v))
    dv_new = fmaf((omega * inv_v).astype(F), t, (omo * dv).astype(F))
    m = ((ii + jj) % 2) == is_black
    return np.where(m, du_new, du).astype(F), np.where(m, dv_new, dv).astype(F)


def calc(I0: np.ndarray, I1: np.ndarray, P: BroxParams | None = None, rsqrt="exact", counters=None) -> np.ndarray:
    """NCVBroxOpticalFlow (NB:598-985) behind BroxOpticalFlowImpl::calc (brox.cpp:129-188).
    I0, I1: float32 in [0, 1].  Returns flow (H, W, 2).  counters: dict, receives COUNTER_NAMES."""
    P = P or BroxParams()
    if rsqrt not in RSQRT_MODES:
        raise ValueError(rsqrt)
    assert I0.dtype == np.float32 and I0.shape == I1.shape
    cnt = dict.fromkeys(COUNTER_NAMES, 0)
    h, w = I0.shape
    sizes = pyramid_sizes(h, w, P.scale_factor, P.outer_iterations)
    pyr0, pyr1 = [I0], [I1]
    inv_sf = F(1.0) / F(P.scale_factor)
    for (lh, lw) in sizes[1:]:
        pyr0.append(resize_supersample(pyr0[-1], lh, lw, inv_sf, cnt))
        pyr1.append(resize_supersample(pyr1[-1], lh, lw, inv_sf))
    lh, lw = sizes[-1]
    u = np.zeros((lh, lw), F)
    v = np.zeros((lh, lw), F)
    for lvl in range(len(sizes) - 1, -1, -1):
        A, B = pyr0[lvl], pyr1[lvl]
        du = np.zeros_like(u)
        dv = np.zeros_like(v)
        Ix0, Iy0 = filter5(A, 1), filter5(A, 0)
        Ix, Iy = filter5(B, 1), filter5(B, 0)
        Ixx, Iyy, Ixy = filter5(Ix, 1), filter5(Iy, 0), filter5(Iy, 1)
        W = warp_terms(u, v, A, B, Ix, Ixx, Ix0, Iy, Iyy, Iy0, Ixy, cnt)
        for inner in range(P.inner_iterations):
            sx, sy, inv_u, inv_v, num_dudv, num_u, num_v = prepare_sor(u, v, du, dv, W, P.alpha, P.gamma, rsqrt,
                                                                         lvl, inner)
            for _ in range(P.solver_iterations):
                du, dv = sor_pass(0, u, v, du, dv, sx, sy, inv_u, inv_v, num_u, num_v, num_dudv)
                du, dv = sor_pass(1, u, v, du, dv, sx, sy, inv_u, inv_v, num_u, num_v, num_dudv)
        u = (u + du).astype(F)
        v = (v + dv).astype(F)
        cnt["levels"] += 1
        if lvl > 0:
            nh, nw = sizes[lvl - 1]
            s = F(1.0) / inv_sf  # kernel gets 1/xFactor with xFactor = 1/scale_factor  (NB:952-953, NS:2270)
            u = resize_bicubic(u, nh, nw, s, inv_sf)
            v = resize_bicubic(v, nh, nw, s, inv_sf)
    if counters is not None:
        counters.update(cnt)
    return np.stack([u, v], axis=-1)
