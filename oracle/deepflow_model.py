"""numpy model of the DeepFlow engine (opencv_contrib_b200/csrc/deepflow.cu): the optflow module's DeepFlow driver
(modules/optflow/src/deepflow.cpp) around a restatement of ``cv::VariationalRefinement`` (opencv's video module).

TEST INFRASTRUCTURE (see oracle/__init__.py).  The source of VariationalRefinement is not restated from anywhere: its
discretization was established by probing ``cv2.VariationalRefinement`` (single calls, 1 fixed-point iteration, 0-2
SOR iterations, ramps, noise and impulses, zero and non-zero initial flow), and tests/test_deepflow_model_cpu.py pins
it against the live cv2 per call.  What it computes on a level, given the flow (u, v):

* I1 warped by ``remap(INTER_LINEAR, BORDER_REPLICATE)`` at (x + u, y + v): coordinates rounded (half to even) to 1/32
  pixel, exact 1/32 weights, taps clamped to the image;
* avg = 0.5 I0 + 0.5 warped I1;  Ix, Iy = undivided central differences of avg (replicated border);  Iz = warped I1 - I0;
  Ixx, Ixy = differences of Ix along x, y;  Iyy of Iy;  Ixz, Iyz of Iz;
* per fixed-point step, with the increment (du, dv) of this call (zero at the start):
  - colour constancy, normalised by |grad I|^2 + zeta^2 (zeta 0.1), robust weight (delta / 2) / sqrt(q^2 / n + eps^2)
    (eps 0.001), q = Iz + Ix du + Iy dv; zeta^2 added to A11 and A22;
  - gradient constancy likewise with weight (gamma / 2) / sqrt(qx^2 / n1 + qy^2 / n2 + eps^2);
  - smoothness: one weight per pixel, (alpha / 2) / sqrt(ux^2 + vx^2 + uy^2 + vy^2 + eps^2) from forward differences
    of (u + du, v + dv) (zero at the far edge), used for the edge to the right and the edge below (zero at the far
    edge); the edges' terms towards (u, v) go to the right-hand side;
  - red-black SOR with omega, the cells with even x + y first, du then dv (dv's coupling uses the new du);
* u += du, v += dv.

Rounding: ``dtype=np.float32`` rounds every operation once, in the order written here; the engine is compiled without
multiply-add contraction (``-fmad=false``) and evaluates the same expressions in the same order, so the two agree bit
for bit.  ``dtype=np.float64`` is the yardstick: the float32 model's distance to it is the rounding noise any float32
implementation carries, and the per-call bound against cv2 is a small multiple of it.
"""
from __future__ import annotations

import math

import numpy as np

from .deepflow_ref import DeepFlowParams, float_sigma, kernel_len, pyramid_sizes, solver_params

ZETA = 0.1
EPSILON = 0.001


def gaussian_taps(sigma: float, ksize: int = 3) -> tuple[float, float]:
    """(centre, side) taps of getGaussianKernel(3, sigma, CV_32F) for the reference's float sigma: computed in double,
    normalised, stored as float."""
    if ksize != 3:
        raise ValueError("the engine's pre-smoothing is the 3-tap kernel (sigma < 1)")
    sigma = float_sigma(sigma)
    t = [math.exp(-0.5 / (sigma * sigma) * (i - 1.0) ** 2) for i in range(3)]
    s = 1.0 / sum(t)
    return float(np.float32(t[1] * s)), float(np.float32(t[0] * s))


def _reflect101(i, n):
    i = np.where(i < 0, -i, i)
    i = np.where(i >= n, 2 * n - 2 - i, i)
    return np.clip(i, 0, n - 1)


def blur3(img, k0, k1, dt=np.float32):
    """3x3 separable Gaussian, reflect-101 border: rows k0 x + k1 (l + r), then the same down the columns."""
    a = img.astype(dt)
    k0, k1 = dt(k0), dt(k1)
    h, w = a.shape
    xs = np.arange(w)
    l, r = _reflect101(xs - 1, w), _reflect101(xs + 1, w)
    t = k0 * a + k1 * (a[:, l] + a[:, r])
    ys = np.arange(h)
    d, u = _reflect101(ys - 1, h), _reflect101(ys + 1, h)
    return (k0 * t + k1 * (t[d, :] + t[u, :])).astype(dt)


def _resize_axis(n_src, n_dst):
    """cv::resize INTER_LINEAR source index and fraction per destination index (centre-aligned, clamped)."""
    scale = n_src / n_dst  # double, as resize.cpp computes 1 / inv_scale
    i0, fr = [], []
    for d in range(n_dst):
        f = np.float32((d + 0.5) * scale - 0.5)
        s = math.floor(f)
        f = np.float32(f - np.float32(s))
        if s < 0:
            s, f = 0, np.float32(0)
        if s >= n_src - 1:
            s, f = n_src - 1, np.float32(0)
        i0.append(s)
        fr.append(f)
    i0 = np.array(i0)
    return i0, np.minimum(i0 + 1, n_src - 1), np.array(fr, np.float32)


def resize_linear(src, rows, cols, mul=None, dt=np.float32):
    """cv::resize(INTER_LINEAR) of a float plane: horizontal pass s0 (1 - fx) + s1 fx, then vertical the same;
    optionally times ``mul`` (the flow prolongation's 1 / 0.95f)."""
    a = src.astype(dt)
    h, w = a.shape
    x0, x1, fx = _resize_axis(w, cols)
    y0, y1, fy = _resize_axis(h, rows)
    fx, fy = fx.astype(dt), fy.astype(dt)
    one = dt(1)
    t = a[:, x0] * (one - fx) + a[:, x1] * fx
    out = t[y0, :] * (one - fy)[:, None] + t[y1, :] * fy[:, None]
    if mul is not None:
        out = out * dt(mul)
    return out.astype(dt)


def _edge(a, axis, step):
    """a shifted by `step` along `axis` with the border replicated (a[clamp(i + step)])."""
    n = a.shape[axis]
    idx = np.clip(np.arange(n) + step, 0, n - 1)
    return np.take(a, idx, axis=axis)


def warp_terms(I0, I1, u, v, dt=np.float32):
    """The planes the data term needs: Ix, Iy, Iz, Ixx, Ixy, Iyy, Ixz, Iyz (VariationalRefinement's prepareBuffers)."""
    h, w = I0.shape
    I0 = I0.astype(dt)
    I1 = I1.astype(dt)
    ys, xs = np.mgrid[0:h, 0:w]
    mx = (xs.astype(np.float32) + u.astype(np.float32)).astype(np.float32)
    my = (ys.astype(np.float32) + v.astype(np.float32)).astype(np.float32)
    X = np.rint(mx * np.float32(32)).astype(np.int64)
    Y = np.rint(my * np.float32(32)).astype(np.int64)
    x0, y0 = X >> 5, Y >> 5
    fx = ((X & 31).astype(np.float32) * np.float32(1 / 32)).astype(dt)
    fy = ((Y & 31).astype(np.float32) * np.float32(1 / 32)).astype(dt)
    xa, xb = np.clip(x0, 0, w - 1), np.clip(x0 + 1, 0, w - 1)
    ya, yb = np.clip(y0, 0, h - 1), np.clip(y0 + 1, 0, h - 1)
    one = dt(1)
    # exact weights (multiples of 1/1024); summed left to right
    w00, w01, w10, w11 = (one - fy) * (one - fx), (one - fy) * fx, fy * (one - fx), fy * fx
    wI = I1[ya, xa] * w00 + I1[ya, xb] * w01 + I1[yb, xa] * w10 + I1[yb, xb] * w11
    avg = dt(0.5) * I0 + dt(0.5) * wI
    dx = lambda a: _edge(a, 1, 1) - _edge(a, 1, -1)
    dy = lambda a: _edge(a, 0, 1) - _edge(a, 0, -1)
    Ix, Iy, Iz = dx(avg), dy(avg), wI - I0
    return dict(Ix=Ix, Iy=Iy, Iz=Iz, Ixx=dx(Ix), Ixy=dy(Ix), Iyy=dy(Iy), Ixz=dx(Iz), Iyz=dy(Iz))


def system_terms(T, u, v, du, dv, alpha, delta, gamma, dt=np.float32):
    """One fixed-point step's linear system: a12, b1, b2, den_u = a11 + sum of edge weights, den_v, and the edge weights
    wr (to the right) and wd (below)."""
    z2 = dt(dt(ZETA) * dt(ZETA))
    e2 = dt(dt(EPSILON) * dt(EPSILON))
    delta2, gamma2, alpha2 = dt(dt(delta) * dt(0.5)), dt(dt(gamma) * dt(0.5)), dt(dt(alpha) * dt(0.5))
    Ix, Iy, Iz, Ixx, Ixy, Iyy, Ixz, Iyz = (T[k] for k in ("Ix", "Iy", "Iz", "Ixx", "Ixy", "Iyy", "Ixz", "Iyz"))
    # colour constancy
    n = Ix * Ix + Iy * Iy + z2
    q = Iz + Ix * du + Iy * dv
    wt = delta2 / np.sqrt(q * q / n + e2) / n
    a11 = wt * (Ix * Ix) + z2
    a12 = wt * (Ix * Iy)
    a22 = wt * (Iy * Iy) + z2
    b1 = -(wt * (Iz * Ix))
    b2 = -(wt * (Iz * Iy))
    # gradient constancy
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
    # smoothness
    U, V = u + du, v + dv
    ux, vx = _edge(U, 1, 1) - U, _edge(V, 1, 1) - V
    uy, vy = _edge(U, 0, 1) - U, _edge(V, 0, 1) - V
    s = alpha2 / np.sqrt(ux * ux + vx * vx + uy * uy + vy * vy + e2)
    wr, wd = s.copy(), s.copy()
    wr[:, -1] = 0
    wd[-1, :] = 0
    wl, wu = _edge(wr, 1, -1), _edge(wd, 0, -1)
    wl[:, 0] = 0
    wu[0, :] = 0
    def div(a):
        return (wr * (_edge(a, 1, 1) - a) + wl * (_edge(a, 1, -1) - a) + wd * (_edge(a, 0, 1) - a) +
                wu * (_edge(a, 0, -1) - a))
    b1 = b1 + div(u)
    b2 = b2 + div(v)
    S = wr + wl + wd + wu
    return dict(a12=a12, b1=b1, b2=b2, den_u=a11 + S, den_v=a22 + S, wr=wr, wd=wd)


def sor(S, du, dv, omega, iterations, dt=np.float32):
    """`iterations` red-black SOR iterations (cells with even x + y first)."""
    h, w = du.shape
    om = dt(omega)
    omo = dt(dt(1) - om)
    wr, wd = S["wr"], S["wd"]
    wl, wu = _edge(wr, 1, -1), _edge(wd, 0, -1)
    wl[:, 0] = 0
    wu[0, :] = 0
    ys, xs = np.mgrid[0:h, 0:w]
    red = ((xs + ys) & 1) == 0
    def nb(a):
        return wr * _edge(a, 1, 1) + wl * _edge(a, 1, -1) + wd * _edge(a, 0, 1) + wu * _edge(a, 0, -1)
    du, dv = du.copy(), dv.copy()
    for _ in range(iterations):
        for colour in (red, ~red):
            ndu = omo * du + om * (S["b1"] + nb(du) - S["a12"] * dv) / S["den_u"]
            du = np.where(colour, ndu, du)
            ndv = omo * dv + om * (S["b2"] + nb(dv) - S["a12"] * du) / S["den_v"]
            dv = np.where(colour, ndv, dv)
    return du, dv


def refine(I0, I1, u, v, alpha, delta, gamma, omega, fixed_point_iterations, sor_iterations, dt=np.float32,
           trace=None):
    """One VariationalRefinement::calcUV call; returns (u, v).  ``trace`` (a list) receives every stage's planes."""
    u, v = u.astype(dt), v.astype(dt)
    T = warp_terms(I0, I1, u, v, dt)
    if trace is not None:
        trace.append(("warp", T))
    du = np.zeros_like(u)
    dv = np.zeros_like(v)
    for _ in range(fixed_point_iterations):
        S = system_terms(T, u, v, du, dv, alpha, delta, gamma, dt)
        if trace is not None:
            trace.append(("terms", S))
        du, dv = sor(S, du, dv, omega, sor_iterations, dt)
        if trace is not None:
            trace.append(("sor", (du, dv)))
    return u + du, v + dv


def model_solver(dt=np.float32):
    """A per-level solver for oracle.deepflow_ref.calc built from this model."""
    def solve(I0, I1, flow, sp):
        u, v = refine(I0, I1, flow[..., 0], flow[..., 1], sp["alpha"], sp["delta"], sp["gamma"], sp["omega"],
                      sp["fixed_point_iterations"], sp["sor_iterations"], dt)
        return np.stack([u, v], axis=-1)
    return solve


def calc(I0, I1, p: DeepFlowParams = DeepFlowParams(), dt=np.float32):
    """The engine's whole pair: pre-smoothing, pyramid, per-level refinement, prolongation; (h, w, 2)."""
    if kernel_len(p.sigma) != 3:
        raise ValueError("the engine's pre-smoothing is the 3-tap kernel (sigma < 1)")
    k0, k1 = gaussian_taps(p.sigma)
    a = blur3(I0.astype(np.float32), k0, k1, dt)
    b = blur3(I1.astype(np.float32), k0, k1, dt)
    sizes = pyramid_sizes(*a.shape, p)
    pyr0, pyr1 = [a], [b]
    for r, c in sizes[1:]:
        pyr0.append(resize_linear(pyr0[-1], r, c, dt=dt))
        pyr1.append(resize_linear(pyr1[-1], r, c, dt=dt))
    sp = solver_params(p)
    r, c = sizes[-1]
    u = np.zeros((r, c), dt)
    v = np.zeros((r, c), dt)
    mul = np.float32(np.float32(1.0) / np.float32(p.downscale_factor))
    for i in range(len(sizes) - 1, -1, -1):
        if i < len(sizes) - 1:
            r, c = sizes[i]
            u = resize_linear(u, r, c, mul, dt)
            v = resize_linear(v, r, c, mul, dt)
        u, v = refine(pyr0[i], pyr1[i], u, v, sp["alpha"], sp["delta"], sp["gamma"], sp["omega"],
                      sp["fixed_point_iterations"], sp["sor_iterations"], dt)
    return np.stack([u, v], axis=-1).astype(np.float32)
