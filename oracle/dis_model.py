"""numpy model of the DIS engine (opencv_contrib_b200/csrc/dis.cu): ``cv::DISOpticalFlow`` (opencv's video module,
dense inverse search) with the spatial propagation of its OpenCL formulation.

TEST INFRASTRUCTURE (see oracle/__init__.py).  What it computes for a u8 pair:

* **Pyramid.**  Level ``finest`` is ``resize(INTER_AREA)`` of the frame to ``(rows >> finest, cols >> finest)``
  (integer division at each halving), every coarser level the same of the level below it: at exact halves the
  rounded box mean ``(a + b + c + d + 2) >> 2``, otherwise OpenCV's general area filter (float weights, rows summed
  with float accumulation, rounded half to even).  The coarsest level is ``min(coarsest, auto)`` where ``auto =
  min(int(log2(max(rows, cols) / (4 ps)) + 0.5), int(log2(min(rows, cols) // ps)))``; a negative ``coarsest`` means
  ``auto``.
* **Per level**, coarse to fine: 3x3 Sobel gradients (int16, reflect-101); per patch (``ps`` = 8, ``stride``; the grid
  ``ws = 1 + (w - ps) // stride`` by ``hs``) the structure-tensor sums xx, yy, xy, x, y as the exact integer sums
  rounded once to float; the patch flows initialised from the dense flow at each patch's centre; with spatial
  propagation a forward scan along each patch row (keep the carried flow when its SSD is lower than the patch's own),
  a descent of every patch, a backward scan (take the right neighbour's flow when its SSD is lower), a second
  descent; without it, one descent.  Then densification (``1 / max(1, |err|)`` weights), the variational refinement
  (deepflow_model's system with DIS's epsilon) and prolongation (``resize`` INTER_LINEAR times 2).
* **Descent** (inverse compositional, ``gd`` iterations): I1 is sampled bilinearly from the level extended by 16
  replicated pixels; the patch's 64 differences are summed per row left to right, the 8 row sums as
  ``((r0 + r4) + (r2 + r6)) + ((r1 + r5) + (r3 + r7))``; the flow steps by the inverse structure tensor
  (``|det| < 1e-3`` takes ``1 / 1e-3``), stops after the step that did not lower the SSD, and a result farther than
  ``ps`` from the start is dropped.
* **Output**: the finest level's flow resized to the frame (INTER_LINEAR) times ``2^finest``.  The search starts from
  zero flow on the coarsest level; the caller's flow is not read.

Spatial propagation is the OpenCL kernels' (dis_flow.cpp's ocl path): all patch rows scan independently and every
patch descends from the scan's pick.  The CPU path that cv2 runs interleaves propagation and descent patch by patch,
so with propagation on the engine and cv2 agree statistically, not bit for bit.

Rounding: ``dtype=np.float32`` rounds every operation once in the order stated; the engine is compiled with
``-fmad=false`` and evaluates the same expressions in the same order, so the two agree bit for bit.
``dtype=np.float64`` is the rounding yardstick.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from . import deepflow_model as dfm

BORDER = 16
EPS = 0.001
PRESET_ULTRAFAST, PRESET_FAST, PRESET_MEDIUM = 0, 1, 2
# per preset, (median, 99th percentile) of the endpoint difference between this model and cv2 4.13 (propagation on) on
# the 640x480 / 1080p smooth-motion pairs of oracle.synth, seed 1: the yardstick of the statistical tests
CV2_MEASURED = {PRESET_ULTRAFAST: (0.033, 0.15), PRESET_FAST: (0.0133, 0.056), PRESET_MEDIUM: (0.0057, 0.035)}


@dataclasses.dataclass(frozen=True)
class DISParams:
    """``cv::DISOpticalFlow``'s settings; the defaults are the FAST preset."""
    finest_scale: int = 2
    coarsest_scale: int = -1
    patch_size: int = 8
    patch_stride: int = 4
    grad_descent_iterations: int = 16
    variational_refinement_iterations: int = 5
    alpha: float = 20.0
    delta: float = 5.0
    gamma: float = 10.0
    epsilon: float = 0.01
    use_mean_normalization: bool = True
    use_spatial_propagation: bool = True


def preset(p: int) -> DISParams:
    """``DISOpticalFlow::create(preset)``."""
    if p == PRESET_ULTRAFAST:
        return DISParams(grad_descent_iterations=12, variational_refinement_iterations=0)
    if p == PRESET_FAST:
        return DISParams()
    if p == PRESET_MEDIUM:
        return DISParams(finest_scale=1, patch_stride=3, grad_descent_iterations=25)
    raise ValueError(p)


def auto_coarsest(rows: int, cols: int, ps: int) -> int:
    return min(int(math.log(max(rows, cols) / (4.0 * ps)) / math.log(2.0) + 0.5),
               int(math.log(min(rows, cols) // ps) / math.log(2.0)) if min(rows, cols) >= ps else -1)


def level_sizes(rows: int, cols: int, p: DISParams) -> list[tuple[int, int]]:
    """(rows, cols) of levels finest .. coarsest."""
    c = auto_coarsest(rows, cols, p.patch_size)
    if p.coarsest_scale >= 0:
        c = min(c, p.coarsest_scale)
    if c < p.finest_scale:
        raise ValueError("the frame is too small for the finest scale")
    sizes = [(rows >> p.finest_scale, cols >> p.finest_scale)]
    for _ in range(p.finest_scale, c):
        sizes.append((sizes[-1][0] // 2, sizes[-1][1] // 2))
    return sizes


def _area_tab(n_src: int, n_dst: int):
    """OpenCV's computeResizeAreaTab for one axis: per destination index a list of (source index, float weight)."""
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
            t.append((s1 - 1, np.float32((s1 - f1) / cw)))
        for s in range(s1, s2):
            t.append((s, np.float32(1.0 / cw)))
        if f2 - s2 > 1e-3:
            t.append((s2, np.float32(min(min(f2 - s2, 1.0), cw) / cw)))
        tab.append(t)
    return tab


def resize_area_u8(src: np.ndarray, rows: int, cols: int) -> np.ndarray:
    """cv::resize(INTER_AREA) of a u8 plane to about half its size."""
    h, w = src.shape
    if h == 2 * rows and w == 2 * cols:
        s = src.astype(np.int32)
        return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    xt, yt = _area_tab(w, cols), _area_tab(h, rows)
    f = src.astype(np.float32)
    # per source row: buf[dx] = sum over the x tab of src * alpha, from 0
    buf = np.zeros((h, cols), np.float32)
    for dx, t in enumerate(xt):
        acc = np.zeros(h, np.float32)
        for sx, a in t:
            acc = acc + f[:, sx] * a
        buf[:, dx] = acc
    out = np.zeros((rows, cols), np.float32)
    for dy, t in enumerate(yt):
        acc = None
        for sy, b in t:
            acc = b * buf[sy] if acc is None else acc + b * buf[sy]
        out[dy] = acc
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def pyramid(I: np.ndarray, sizes) -> list[np.ndarray]:
    out = []
    src = I
    for r, c in sizes:
        src = resize_area_u8(src, r, c) if (r, c) != src.shape else src.copy()
        out.append(src)
    return out


def sobel(I: np.ndarray):
    """cv::spatialGradient: 3x3 Sobel, reflect-101 border, int16 (returned as int32)."""
    p = np.pad(I.astype(np.int32), 1, mode="reflect")
    gx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    gy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    return gx, gy


def grid(h: int, w: int, ps: int, stride: int) -> tuple[int, int]:
    """(hs, ws): patches per column and per row."""
    return 1 + (h - ps) // stride, 1 + (w - ps) // stride


def structure_tensor(gx, gy, ps, stride, dt=np.float32):
    """Per patch xx, yy, xy, x, y: exact integer sums over the patch, rounded once."""
    h, w = gx.shape
    hs, ws = grid(h, w, ps, stride)
    def box(a):
        c = np.zeros((h + 1, w + 1), np.int64)
        c[1:, 1:] = a.astype(np.int64).cumsum(0).cumsum(1)
        i = np.arange(hs)[:, None] * stride
        j = np.arange(ws)[None, :] * stride
        return (c[i + ps, j + ps] - c[i, j + ps] - c[i + ps, j] + c[i, j]).astype(dt)
    return dict(xx=box(gx * gx), yy=box(gy * gy), xy=box(gx * gy), x=box(gx), y=box(gy))


class _Level:
    """One level's images and the patch evaluation shared by the scans and the descent."""

    def __init__(self, I0, I1, ps, stride, mean_norm, dt):
        self.dt = dt
        self.h, self.w = I0.shape
        self.ps, self.stride, self.mean_norm = ps, stride, mean_norm
        self.I0 = I0.astype(dt)
        self.I1e = np.pad(I1, BORDER, mode="edge").astype(dt)
        gx, gy = sobel(I0)
        self.gx, self.gy = gx.astype(dt), gy.astype(dt)
        self.T = structure_tensor(gx, gy, ps, stride, dt)
        self.hs, self.ws = grid(self.h, self.w, ps, stride)

    def terms(self, ii, jj, ux, uy, grads):
        """For patches with top-left (ii, jj) at flows (ux, uy): (sum diff, sum diff^2[, sum diff Ix, sum diff Iy])."""
        dt, ps = self.dt, self.ps
        one, b = dt(1), dt(BORDER)
        yI = np.minimum(np.maximum((ii.astype(dt) + uy) + b, dt(BORDER - ps + 1)), dt(BORDER + self.h - 1))
        xI = np.minimum(np.maximum((jj.astype(dt) + ux) + b, dt(BORDER - ps + 1)), dt(BORDER + self.w - 1))
        di, dj = yI - np.floor(yI), xI - np.floor(xI)
        w11, w10, w01, w00 = di * dj, di * (one - dj), (one - di) * dj, (one - di) * (one - dj)
        r0, c0 = yI.astype(np.int64), xI.astype(np.int64)
        a9 = np.arange(ps + 1)
        win = self.I1e[r0[:, None, None] + a9[None, :, None], c0[:, None, None] + a9[None, None, :]]
        a8 = np.arange(ps)
        ri, ci = ii[:, None, None] + a8[None, :, None], jj[:, None, None] + a8[None, None, :]
        W = lambda x: x[:, None, None]
        d = (((W(w00) * win[:, :ps, :ps] + W(w01) * win[:, :ps, 1:]) + W(w10) * win[:, 1:, :ps]) +
             W(w11) * win[:, 1:, 1:]) - self.I0[ri, ci]
        planes = [d, d * d]
        if grads:
            planes += [d * self.gx[ri, ci], d * self.gy[ri, ci]]
        return [self._reduce(p) for p in planes]

    @staticmethod
    def _reduce(p):
        r = p[:, :, 0]
        for c in range(1, p.shape[2]):
            r = r + p[:, :, c]
        return ((r[:, 0] + r[:, 4]) + (r[:, 2] + r[:, 6])) + ((r[:, 1] + r[:, 5]) + (r[:, 3] + r[:, 7]))

    def ssd(self, ii, jj, ux, uy):
        sd, sq = self.terms(ii, jj, ux, uy, False)
        if self.mean_norm:
            return sq - (sd * sd) * self.dt(1.0 / (self.ps * self.ps))
        return sq

    def descent(self, Sx, Sy, iters):
        """Every patch from (Sx, Sy): ``iters`` inverse-compositional steps; returns the new (Sx, Sy)."""
        dt = self.dt
        ii, jj = (a.ravel() * self.stride for a in np.mgrid[0:self.hs, 0:self.ws])
        k = np.arange(ii.size)
        xx, yy, xy = (self.T[n].ravel() for n in ("xx", "yy", "xy"))
        xs, ys = self.T["x"].ravel(), self.T["y"].ravel()
        det = xx * yy - xy * xy
        inv = np.where(np.abs(det) < dt(EPS), dt(1) / dt(EPS), dt(1) / np.where(det == 0, dt(1), det)).astype(dt)
        h11, h12, h22 = yy * inv, (-xy) * inv, xx * inv
        U0x, U0y = Sx.ravel().copy(), Sy.ravel().copy()
        cx, cy = U0x.copy(), U0y.copy()
        prev = np.full(ii.size, dt(1e10), dt)
        inv_n = dt(1.0 / (self.ps * self.ps))
        for _ in range(iters):
            if k.size == 0:
                break
            sd, sq, gx, gy = self.terms(ii[k], jj[k], cx[k], cy[k], True)
            if self.mean_norm:
                ssd = sq - (sd * sd) * inv_n
                dux = gx - (sd * xs[k]) * inv_n
                duy = gy - (sd * ys[k]) * inv_n
            else:
                ssd, dux, duy = sq, gx, gy
            cx[k] = cx[k] - (h11[k] * dux + h12[k] * duy)
            cy[k] = cy[k] - (h12[k] * dux + h22[k] * duy)
            go = ssd < prev[k]
            prev[k] = ssd
            k = k[go]
        vx, vy = cx - U0x, cy - U0y
        ok = (vx * vx + vy * vy) <= dt(self.ps * self.ps)
        return np.where(ok, cx, U0x).reshape(self.hs, self.ws), np.where(ok, cy, U0y).reshape(self.hs, self.ws)

    def scan_forward(self, Sx, Sy):
        """Each patch row scanned left to right from the patches' own start flows (Sx, Sy)."""
        ii = np.arange(self.hs) * self.stride
        Sx, Sy = Sx.copy(), Sy.copy()
        px, py = Sx[:, 0].copy(), Sy[:, 0].copy()
        for js in range(1, self.ws):
            jj = np.full(self.hs, js * self.stride)
            own = self.ssd(ii, jj, Sx[:, js], Sy[:, js])
            car = self.ssd(ii, jj, px, py)
            keep = car < own
            px, py = np.where(keep, px, Sx[:, js]), np.where(keep, py, Sy[:, js])
            Sx[:, js], Sy[:, js] = px, py
        return Sx, Sy

    def scan_backward(self, Sx, Sy):
        ii = np.arange(self.hs) * self.stride
        Sx, Sy = Sx.copy(), Sy.copy()
        for js in range(self.ws - 2, -1, -1):
            jj = np.full(self.hs, js * self.stride)
            own = self.ssd(ii, jj, Sx[:, js], Sy[:, js])
            right = self.ssd(ii, jj, Sx[:, js + 1], Sy[:, js + 1])
            take = right < own
            Sx[:, js] = np.where(take, Sx[:, js + 1], Sx[:, js])
            Sy[:, js] = np.where(take, Sy[:, js + 1], Sy[:, js])
        return Sx, Sy

    def initial(self, Ux, Uy, zero_candidate=False):
        """Each patch's start: the dense flow at its centre; with ``zero_candidate`` zero flow instead where its SSD is
        lower (cv2 does this on the level that receives the caller's initial flow)."""
        c = self.ps // 2
        i = np.arange(self.hs)[:, None] * self.stride + c
        j = np.arange(self.ws)[None, :] * self.stride + c
        Sx, Sy = Ux[i, j].astype(self.dt), Uy[i, j].astype(self.dt)
        if zero_candidate:
            ii, jj = (a.ravel() * self.stride for a in np.mgrid[0:self.hs, 0:self.ws])
            own = self.ssd(ii, jj, Sx.ravel(), Sy.ravel())
            zero = self.ssd(ii, jj, np.zeros(ii.size, self.dt), np.zeros(ii.size, self.dt))
            z = (zero < own).reshape(self.hs, self.ws)
            Sx, Sy = np.where(z, self.dt(0), Sx), np.where(z, self.dt(0), Sy)
        return Sx, Sy

    def densify(self, Sx, Sy, I0u8, I1u8):
        """Dense flow: the patches covering each pixel, weighted by 1 / max(1, |I1 at the moved pixel - I0|)."""
        dt, h, w, ps, st = self.dt, self.h, self.w, self.ps, self.stride
        I0, I1 = I0u8.astype(dt), I1u8.astype(dt)
        ys, xs = np.mgrid[0:h, 0:w]
        end_i = np.minimum(ys // st, (h - ps) // st)
        start_i = np.minimum(np.maximum(0, ys - ps + st) // st, end_i)
        end_j = np.minimum(xs // st, (w - ps) // st)
        start_j = np.minimum(np.maximum(0, xs - ps + st) // st, end_j)
        su, sv, sc = (np.zeros((h, w), dt) for _ in range(3))
        K = (ps + st - 1) // st + 1
        fx, fy = xs.astype(dt), ys.astype(dt)
        lim_x, lim_y = dt(dt(w) - dt(1)) - dt(EPS), dt(dt(h) - dt(1)) - dt(EPS)
        for a in range(K):
            i_s = start_i + a
            for b in range(K):
                j_s = start_j + b
                m = (i_s <= end_i) & (j_s <= end_j)
                if not m.any():
                    continue
                sx = Sx[np.minimum(i_s, self.hs - 1), np.minimum(j_s, self.ws - 1)]
                sy = Sy[np.minimum(i_s, self.hs - 1), np.minimum(j_s, self.ws - 1)]
                jm = np.minimum(np.maximum(fx + sx, dt(0)), lim_x)
                im = np.minimum(np.maximum(fy + sy, dt(0)), lim_y)
                jl, il = jm.astype(np.int64), im.astype(np.int64)
                ju, iu = jl + 1, il + 1
                fjl, fil, fju, fiu = jl.astype(dt), il.astype(dt), ju.astype(dt), iu.astype(dt)
                diff = ((((jm - fjl) * (im - fil)) * I1[iu, ju] + ((fju - jm) * (im - fil)) * I1[iu, jl]) +
                        ((jm - fjl) * (fiu - im)) * I1[il, ju]) + ((fju - jm) * (fiu - im)) * I1[il, jl] - I0
                coef = dt(1) / np.maximum(dt(1), np.abs(diff))
                su = np.where(m, su + coef * sx, su)
                sv = np.where(m, sv + coef * sy, sv)
                sc = np.where(m, sc + coef, sc)
        return (su / sc).astype(dt), (sv / sc).astype(dt)


def system_terms(T, u, v, du, dv, alpha, delta, gamma, epsilon, dt=np.float32):
    """deepflow_model.system_terms with the robust functions' epsilon as an argument (DeepFlow's is 0.001)."""
    z2 = dt(dt(dfm.ZETA) * dt(dfm.ZETA))
    e2 = dt(dt(epsilon) * dt(epsilon))
    delta2, gamma2, alpha2 = dt(dt(delta) * dt(0.5)), dt(dt(gamma) * dt(0.5)), dt(dt(alpha) * dt(0.5))
    Ix, Iy, Iz, Ixx, Ixy, Iyy, Ixz, Iyz = (T[k] for k in ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz"))
    n = Ix * Ix + Iy * Iy + z2
    q = Iz + Ix * du + Iy * dv
    wt = delta2 / np.sqrt(q * q / n + e2) / n
    a11 = wt * (Ix * Ix) + z2
    a12 = wt * (Ix * Iy)
    a22 = wt * (Iy * Iy) + z2
    b1 = -(wt * (Iz * Ix))
    b2 = -(wt * (Iz * Iy))
    n1 = Ixx * Ixx + Ixy * Ixy + z2
    n2 = Iyy * Iyy + Ixy * Ixy + z2
    qx = Ixz + Ixx * du + Ixy * dv
    qy = Iyz + Ixy * du + Iyy * dv
    wg = gamma2 / np.sqrt(qx * qx / n1 + qy * qy / n2 + e2)
    a11 = a11 + wg * (Ixx * Ixx / n1 + Ixy * Ixy / n2)
    a12 = a12 + wg * (Ixx * Ixy / n1 + Ixy * Iyy / n2)
    a22 = a22 + wg * (Ixy * Ixy / n1 + Iyy * Iyy / n2)
    b1 = b1 - wg * (Ixx * Ixz / n1 + Ixy * Iyz / n2)
    b2 = b2 - wg * (Ixy * Ixz / n1 + Iyy * Iyz / n2)
    U, V = u + du, v + dv
    ux, vx = dfm._edge(U, 1, 1) - U, dfm._edge(V, 1, 1) - V
    uy, vy = dfm._edge(U, 0, 1) - U, dfm._edge(V, 0, 1) - V
    s = alpha2 / np.sqrt(ux * ux + vx * vx + uy * uy + vy * vy + e2)
    wr, wd = s.copy(), s.copy()
    wr[:, -1] = 0
    wd[-1, :] = 0
    wl, wu = dfm._edge(wr, 1, -1), dfm._edge(wd, 0, -1)
    wl[:, 0] = 0
    wu[0, :] = 0
    def div(a):
        return (wr * (dfm._edge(a, 1, 1) - a) + wl * (dfm._edge(a, 1, -1) - a) + wd * (dfm._edge(a, 0, 1) - a) +
                wu * (dfm._edge(a, 0, -1) - a))
    b1 = b1 + div(u)
    b2 = b2 + div(v)
    S = wr + wl + wd + wu
    return dict(a12=a12, b1=b1, b2=b2, den_u=a11 + S, den_v=a22 + S, wr=wr, wd=wd)


def refine(I0, I1, u, v, alpha, delta, gamma, epsilon, omega, fixed_point_iterations, sor_iterations, dt=np.float32):
    """deepflow_model.refine (one VariationalRefinement::calcUV call) with epsilon as an argument."""
    u, v = u.astype(dt), v.astype(dt)
    T = dfm.warp_terms(I0, I1, u, v, dt)
    du, dv = np.zeros_like(u), np.zeros_like(v)
    for _ in range(fixed_point_iterations):
        S = system_terms(T, u, v, du, dv, alpha, delta, gamma, epsilon, dt)
        du, dv = dfm.sor(S, du, dv, omega, sor_iterations, dt)
    return u + du, v + dv


REFINE_OMEGA = 1.6
REFINE_SOR_ITERATIONS = 5


def calc_level(I0, I1, Ux, Uy, p: DISParams, dt=np.float32, trace=None, zero_candidate=False):
    """One level: patch search, densification and refinement from the dense flow (Ux, Uy) of the level's size."""
    L = _Level(I0, I1, p.patch_size, p.patch_stride, p.use_mean_normalization, dt)
    Sx, Sy = L.initial(Ux, Uy, zero_candidate)
    if p.use_spatial_propagation:
        Sx, Sy = L.scan_forward(Sx, Sy)
        Sx, Sy = L.descent(Sx, Sy, p.grad_descent_iterations)
        Sx, Sy = L.scan_backward(Sx, Sy)
        Sx, Sy = L.descent(Sx, Sy, p.grad_descent_iterations)
    else:
        Sx, Sy = L.descent(Sx, Sy, p.grad_descent_iterations)
    if trace is not None:
        trace.append(("patches", Sx, Sy))
    ux, uy = L.densify(Sx, Sy, I0, I1)
    if trace is not None:
        trace.append(("dense", ux, uy))
    if p.variational_refinement_iterations > 0:
        ux, uy = refine(I0.astype(np.float32), I1.astype(np.float32), ux, uy, p.alpha, p.delta, p.gamma, p.epsilon,
                        REFINE_OMEGA, p.variational_refinement_iterations, REFINE_SOR_ITERATIONS, dt)
    return ux.astype(dt), uy.astype(dt)


def calc(I0, I1, p: DISParams = DISParams(), dt=np.float32, trace=None, flow=None):
    """The engine's whole pair; (h, w, 2) float32.  ``flow`` (h, w, 2) is the caller's initial flow: resized
    (INTER_LINEAR) to the coarsest level times 1 / 2^coarsest, and on that level each patch starts from it or from
    zero flow, whichever has the lower SSD.  Without it the coarsest level starts from zero."""
    if I0.dtype != np.uint8 or I1.dtype != np.uint8 or I0.shape != I1.shape:
        raise ValueError("DIS takes two u8 frames of one size")
    sizes = level_sizes(*I0.shape, p)
    P0, P1 = pyramid(I0, sizes), pyramid(I1, sizes)
    r, c = sizes[-1]
    if flow is None:
        Ux, Uy = np.zeros((r, c), dt), np.zeros((r, c), dt)
    else:
        m = np.float32(1.0 / (1 << (p.finest_scale + len(sizes) - 1)))
        Ux = dfm.resize_linear(flow[..., 0], r, c, m, dt)
        Uy = dfm.resize_linear(flow[..., 1], r, c, m, dt)
    for k in range(len(sizes) - 1, -1, -1):
        if k < len(sizes) - 1:
            r, c = sizes[k]
            Ux = dfm.resize_linear(Ux, r, c, np.float32(2), dt)
            Uy = dfm.resize_linear(Uy, r, c, np.float32(2), dt)
        Ux, Uy = calc_level(P0[k], P1[k], Ux, Uy, p, dt, trace, flow is not None and k == len(sizes) - 1)
    h, w = I0.shape
    m = np.float32(1 << p.finest_scale)
    return np.stack([dfm.resize_linear(Ux, h, w, m, dt), dfm.resize_linear(Uy, h, w, m, dt)], -1).astype(np.float32)
