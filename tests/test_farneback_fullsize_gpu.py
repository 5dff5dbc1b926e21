"""Farneback engine vs its CUDA-semantics model (oracle/farneback_gpu_model.py) at the shapes each fused iteration kernel
is dispatched on and at the benchmark's frame size: levels at and just past n_SM 64x32 tiles (the 512-thread kernel
gives way to the 256-thread one), every column residue mod 4 at more than two waves (float4 and scalar stores, the quad
gather's tail), rows around the vertical pass's 28-row window, images smaller than one tile, every kernel_path /
aux_path variant, the persistent TMA kernel on both sides of its 2 x n_SM threshold, and the generic kernel at every
window size class.

Default knobs, CUDA graph on, a real stream.  Every case first asserts which iteration kernel ran on each level
(getActivePath), so a shape that silently takes another kernel fails instead of passing vacuously.

Tolerances (see DESIGN.md "Parity"): at the 50 %, 99 %, 99.9 % quantiles and the max, the end-point error of the engine
against the float model is at most 4 x that of the float model against the double model on the same input -- float
rounding alone moves the flow that far, and the engine's running box sum and FMA contraction round differently from the
model.  In the shape sweep, the variant and the generic-kernel cases, FLOORS apply wherever they are the larger.
"""
import time

import numpy as np
import pytest

from oracle import metrics, synth, farneback_gpu_model as fm

pytestmark = pytest.mark.gpu

FT_W, FT_H = 64, 32   # tile of the register-blocked iteration kernels
TT = 64               # tile edge of the persistent TMA kernel
WIN = 28              # rows of the vertical pass's register window (FT_H - 4)
FACTOR = 4.0
QUANTILES = (0.5, 0.99, 0.999, 1.0)
FLOORS = {0.5: 2e-6, 0.99: 2e-5, 0.999: 5e-5, 1.0: 2e-4}
ONE_LEVEL = dict(numLevels=0, numIters=3)   # both the update and the final-flow iterations run
BENCH = dict(numLevels=5, winSize=13, numIters=10, polyN=5)


def _check_vs_yardstick(e, yard, floors, label, fails):
    """Quantiles of e = EPE(engine, float model) against FACTOR x the same quantiles of yard = EPE(float model, double
    model); floors: {quantile: bound} applied wherever larger (None: none).  Failures are collected in `fails`."""
    for q in QUANTILES:
        v, y = float(np.quantile(e, q)), float(np.quantile(yard, q))
        bound = max(FACTOR * y, 0.0 if floors is None else floors[q])
        print(f"{label}: q{q:g} engine-vs-f32 {v:.2e}, f32-vs-f64 {y:.2e}, bound {bound:.2e}")
        if not v <= bound:
            fails.append((label, q, v, y, _worst_tiles(e)))


@pytest.fixture(scope="module")
def stream(cuda_device):
    import torch
    return torch.cuda.Stream(device=cuda_device)


@pytest.fixture(scope="module")
def num_sms(cuda_device):
    import torch
    return torch.cuda.get_device_properties(cuda_device).multi_processor_count


def _params(kw):
    return fm.FarnebackParams(**kw)


def _engine(dev, stream, I0, I1, kernel_path=0, aux_path=0, init=None, alg=None, **kw):
    import torch
    import opencv_contrib_b200 as ocb
    if alg is None:
        alg = ocb.FarnebackOpticalFlow_create(**kw)
    alg.setEngineOption("kernel_path", kernel_path)
    alg.setEngineOption("aux_path", aux_path)
    assert alg.getEngineOption("use_graph") == 1 and alg.getEngineOption("fused_iters") == 0
    d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
    fl = None if init is None else torch.from_numpy(np.ascontiguousarray(init)).to(dev)
    f = alg.calc(d0, d1, fl, stream)
    stream.synchronize()
    return f.cpu().numpy(), alg


def _expected_paths(h, w, P, n_sm, kernel_path=0, aux_path=0):
    """The engine's per-level dispatch (FarnebackEngine::solve), restated from the level sizes and the SM count."""
    from opencv_contrib_b200._lib import FARN_PATH
    khalf = P.winSize // 2
    gauss = bool(P.flags & fm.OPTFLOW_FARNEBACK_GAUSSIAN)
    out = []
    for r, c in fm.level_sizes(h, w, P):
        fast6 = khalf == 6 and kernel_path != 1
        wide = -(-c // FT_W) * -(-r // FT_H) <= n_sm
        if P.numIters == 0:
            p = 0
        elif kernel_path == 3 and khalf == 6 and -(-c // TT) * -(-r // TT) >= 2 * n_sm:
            p = FARN_PATH["tma"]
        elif not fast6:
            p = FARN_PATH["generic"]
        elif kernel_path == 2:
            p = FARN_PATH["fast"]
        elif gauss:
            p = FARN_PATH["quad"]
        elif wide:
            p = FARN_PATH["quad_wide"]
        else:
            p = {3: FARN_PATH["quad_r80"], 4: FARN_PATH["quad_r64"], 5: FARN_PATH["quad_transposed"]}.get(
                aux_path, FARN_PATH["quad"])
        out.append(p)
    return out


def _check_paths(alg, h, w, P, n_sm, **knobs):
    want = _expected_paths(h, w, P, n_sm, **knobs)
    got = [alg.getActivePath(s) for s in range(len(want))]
    assert got == want, f"{h}x{w} {knobs}: iteration kernel per level {got}, expected {want}"
    import opencv_contrib_b200 as ocb
    with pytest.raises(ocb.B2FError):
        alg.getActivePath(len(want))   # a level the last calc did not solve
    return got


def _pair(h, w, seed, dtype):
    """A synthetic pair cropped to h x w.  f32: the u8 texture's float values in [0, 255], not rounded to integers
    (the engine converts without scaling, as the reference does)."""
    I0, I1, _ = synth.make_pair(max(h, 16), max(w, 16), seed=seed, kind="smooth", dtype="f32" if dtype == "f32" else "u8")
    if dtype == "f32":
        I0, I1 = I0 * np.float32(255), I1 * np.float32(255)
    return np.ascontiguousarray(I0[:h, :w]), np.ascontiguousarray(I1[:h, :w])


def _worst_tiles(e, n=8):
    """Coordinates of the n worst pixels inside their 64 x 32 tile: a seam defect shows as x mod 64 or y mod 32 at a
    tile edge at every one of them."""
    idx = np.argsort(e, axis=None)[-n:][::-1]
    ys, xs = np.unravel_index(idx, e.shape)
    return [dict(x=int(x), y=int(y), x_mod64=int(x % FT_W), y_mod32=int(y % FT_H), epe=float(e[y, x]))
            for y, x in zip(ys, xs)]


def _models(I0, I1, P, init=None):
    ref = fm.calc(I0, I1, P, init_flow=init)
    yard = metrics.epe(ref, fm.calc(I0, I1, P, init_flow=init, precision="f64"))
    return ref, yard


def _grid(n, rx=29, ry=17):
    """rows, cols of a level with n 64 x 32 tiles (tx * ty == n) and ragged right and bottom edges."""
    tx = max(d for d in range(1, int(n ** 0.5) + 1) if n % d == 0)
    ty = n // tx
    return (ty - 1) * FT_H + ry, (tx - 1) * FT_W + rx


def _sweep_shapes(n_sm):
    """(rows, cols, why, flags): the box window at the tile counts around the 512-thread kernel's limit, both windows
    at every column residue, then the two alternating."""
    shapes = [(*_grid(n), f"{n} tiles", 0) for n in (n_sm, n_sm + 1, 2 * n_sm + 1)]
    ty = 12
    tx = -(-(2 * n_sm + 1) // ty)  # at least 2 n_SM + 1 tiles
    shapes += [((ty - 1) * FT_H + 12, (tx - 1) * FT_W + r, f"cols % 4 == {((tx - 1) * FT_W + r) % 4}, {tx * ty} tiles",
                flags) for r in (29, 30, 31, 32) for flags in (0, 256)]
    small = [(r, 301, "vertical window") for r in (WIN - 1, WIN, WIN + 1, FT_H - 1)]
    small += [(1, 37, "1xN"), (37, 1, "Nx1"), (2, 2, "2x2"), (3, 5, "3x5")]
    return shapes + [(h, w, why, 256 * (i % 2)) for i, (h, w, why) in enumerate(small)]


def test_shape_sweep_vs_model(cuda_device, stream, num_sms):
    """One level, default kernel, box / gaussian, polyN 5 / 7 and u8 / f32 input alternating."""
    t0, fails = time.time(), []
    for i, (h, w, why, flags) in enumerate(_sweep_shapes(num_sms)):
        kw = dict(ONE_LEVEL, flags=flags, **(dict(polyN=7, polySigma=1.5) if i % 4 >= 2 else {}))
        dtype = "f32" if i % 3 == 1 else "u8"
        I0, I1 = _pair(h, w, seed=40 + i, dtype=dtype)
        got, alg = _engine(cuda_device, stream, I0, I1, **kw)
        P = _params(kw)
        paths = _check_paths(alg, h, w, P, num_sms)
        ref, yard = _models(I0, I1, P)
        print(f"sweep {h}x{w} {dtype} {kw} ({why}): active path {paths}")
        assert np.isfinite(got).all()
        _check_vs_yardstick(metrics.epe(got, ref), yard, FLOORS, f"  {h}x{w}", fails)
    print(f"sweep: {time.time() - t0:.1f} s")
    assert not fails, fails


def test_iteration_kernel_variants_vs_model(cuda_device, stream, num_sms):
    """kernel_path 0 / 1 / 2 and aux_path 3 / 4 / 5 at a level past n_SM tiles, box and gaussian, on one handle (each
    change of knob re-captures the graph; the repeat call replays it and must report the same kernels).  aux_path
    3 / 4 / 5 share the summation order of aux_path 0: same bits."""
    h, w = _grid(2 * num_sms + 1)
    fails = []
    for flags in (0, 256):
        kw = dict(ONE_LEVEL, flags=flags)
        P = _params(kw)
        I0, I1 = _pair(h, w, seed=7 + flags, dtype="u8")
        ref, yard = _models(I0, I1, P)
        alg, base = None, None
        for kp, aux in ((0, 0), (1, 0), (2, 0), (0, 3), (0, 4), (0, 5)):
            got, alg = _engine(cuda_device, stream, I0, I1, kernel_path=kp, aux_path=aux, alg=alg, **kw)
            paths = _check_paths(alg, h, w, P, num_sms, kernel_path=kp, aux_path=aux)
            again, _ = _engine(cuda_device, stream, I0, I1, kernel_path=kp, aux_path=aux, alg=alg, **kw)
            assert np.array_equal(again, got) and _check_paths(alg, h, w, P, num_sms, kernel_path=kp,
                                                               aux_path=aux) == paths
            assert np.isfinite(got).all()
            if kp == 0 and aux == 0:
                base = got
            if aux:
                assert np.array_equal(got, base), (flags, aux, float(np.abs(got - base).max()))
            else:
                _check_vs_yardstick(metrics.epe(got, ref), yard, FLOORS,
                                    f"{h}x{w} flags {flags} kernel_path {kp} {paths}", fails)
    assert not fails, fails


def test_persistent_tma_kernel_vs_model(cuda_device, stream, num_sms):
    """kernel_path 3 on levels with at least 2 n_SM + 1 64 x 64 tiles, ragged in both directions, at every column residue
    mod 4 (must run the TMA kernel, equal the default kernel bit for bit and match the model), and on a level just below
    the threshold (must report the fast kernel)."""
    from opencv_contrib_b200._lib import FARN_PATH
    ty = 16
    tx = -(-(2 * num_sms + 1) // ty)
    fails = []
    for i, r in enumerate((29, 30, 31, 32)):
        h, w = (ty - 1) * TT + 23, (tx - 1) * TT + r
        kw = dict(ONE_LEVEL, flags=256 if i % 2 else 0)
        P = _params(kw)
        I0, I1 = _pair(h, w, seed=60 + i, dtype="f32" if i % 2 else "u8")
        got, alg = _engine(cuda_device, stream, I0, I1, kernel_path=3, **kw)
        paths = _check_paths(alg, h, w, P, num_sms, kernel_path=3)
        assert paths[0] == FARN_PATH["tma"]
        dflt, _ = _engine(cuda_device, stream, I0, I1, **kw)
        assert np.array_equal(got, dflt), (h, w, float(np.abs(got - dflt).max()))
        ref, yard = _models(I0, I1, P)
        _check_vs_yardstick(metrics.epe(got, ref), yard, FLOORS, f"tma {h}x{w} cols % 4 == {w % 4} {paths}", fails)
    tx = (2 * num_sms - 1) // ty   # tx * ty < 2 n_SM
    h, w = (ty - 1) * TT + 23, (tx - 1) * TT + 29
    I0, I1 = _pair(h, w, seed=70, dtype="u8")
    _, alg = _engine(cuda_device, stream, I0, I1, kernel_path=3, **ONE_LEVEL)
    paths = _check_paths(alg, h, w, _params(ONE_LEVEL), num_sms, kernel_path=3)
    assert FARN_PATH["tma"] not in paths
    print(f"tma below threshold {h}x{w}: active path {paths}")
    assert not fails, fails


@pytest.mark.parametrize("win", [1, 3, 9, 15, 31])
def test_generic_kernel_window_sizes_vs_model(cuda_device, stream, num_sms, win):
    """k_farn_iter serves every winSize other than 13; winSize 1 is a one-tap window (khalf = 0)."""
    h, w = 300, 700
    fails = []
    for flags in (0, 256):
        kw = dict(ONE_LEVEL, winSize=win, flags=flags)
        P = _params(kw)
        I0, I1 = _pair(h, w, seed=80 + win, dtype="u8")
        got, alg = _engine(cuda_device, stream, I0, I1, **kw)
        paths = _check_paths(alg, h, w, P, num_sms)
        assert np.isfinite(got).all()
        ref, yard = _models(I0, I1, P)
        _check_vs_yardstick(metrics.epe(got, ref), yard, FLOORS, f"winSize {win} flags {flags} {paths}", fails)
    assert not fails, fails


_BENCH_MODELS = {}


def _bench_case(name):
    """Input, parameters and model results of one 1080p case, computed once per module."""
    if name not in _BENCH_MODELS:
        h, w = 1080, 1920
        I0, I1 = _pair(h, w, seed=0, dtype="f32")
        kw, init = dict(BENCH), None
        if name == "gaussian":
            kw["flags"] = fm.OPTFLOW_FARNEBACK_GAUSSIAN
        elif name == "fastPyramids":
            kw["fastPyramids"] = True
        elif name == "initial_flow":
            kw["flags"] = fm.OPTFLOW_USE_INITIAL_FLOW
            yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
            init = np.stack([3.0 * np.sin(xx / 97.0 + yy / 61.0), 2.0 * np.cos(xx / 71.0 - yy / 113.0)], axis=-1)
            init = init.astype(np.float32)
        t0 = time.time()
        ref, yard = _models(I0, I1, _params(kw), init)
        print(f"1080p {name}: model (float + double) {time.time() - t0:.1f} s")
        _BENCH_MODELS[name] = (I0, I1, kw, init, ref, yard)
    return _BENCH_MODELS[name]


@pytest.mark.parametrize("name,kernel_path", [("default", 0), ("default", 3), ("gaussian", 0), ("fastPyramids", 0),
                                              ("initial_flow", 0)])
def test_benchmark_size_vs_model(cuda_device, stream, num_sms, name, kernel_path):
    """1080p with the benchmark's parameters (5 levels, winSize 13, 10 iterations, polyN 5, f32 input)."""
    I0, I1, kw, init, ref, yard = _bench_case(name)
    h, w = I0.shape
    got, alg = _engine(cuda_device, stream, I0, I1, kernel_path=kernel_path, init=init, **kw)
    assert alg.getStats()["levels"] == len(fm.level_sizes(h, w, _params(kw))) == 6
    paths = _check_paths(alg, h, w, _params(kw), num_sms, kernel_path=kernel_path)
    assert np.isfinite(got).all()
    fails = []
    _check_vs_yardstick(metrics.epe(got, ref), yard, None, f"1080p {name} kernel_path {kernel_path} {paths}", fails)
    assert not fails, fails
