"""Farneback engine vs the model of its own roundings (oracle/farneback_model.c, build "eng", through
oracle/farneback_model_native.py), bit for bit, at the shapes each fused iteration kernel is dispatched on and at the
benchmark's frame size: levels at and just past n_SM 64x32 tiles (the 512-thread kernel gives way to the 256-thread
one), every column residue mod 4 at more than two waves (float4 and scalar stores, the quad gather's tail), rows around
the vertical pass's 28-row window and the running box sum's 16-row strips, images smaller than one tile, every
kernel_path / aux_path variant, the persistent TMA kernel on both sides of its 2 x n_SM threshold, the generic kernel at
every window size class, and a ladder of stages that names the first one where engine and model part.

Default knobs, CUDA graph on, a real stream.  Every case first asserts which iteration kernel ran on each level
(getActivePath), so a shape that silently takes another kernel fails instead of passing vacuously.  The model is
computed in the iteration order of the kernel that ran (farneback_model_native.order_for).  Flows are compared as uint32;
NaN is compared by position.  A mismatch reports the count of differing pixels and the first few with their position
inside the 64 x 32 tile, the 4-pixel task and the 16-row strip, where a seam defect shows.
"""
import time

import numpy as np
import pytest

from oracle import synth, farneback_gpu_model as fm, farneback_model_native as fn

pytestmark = pytest.mark.gpu

FT_W, FT_H = 64, 32   # tile of the register-blocked iteration kernels
TT = 64               # tile edge of the persistent TMA kernel
WIN = 28              # rows of the vertical pass's register window (FT_H - 4)
ONE_LEVEL = dict(numLevels=0, numIters=3)   # both the update and the final-flow iterations run
BENCH = dict(numLevels=5, winSize=13, numIters=10, polyN=5)


def _mismatch(got, want, n=6):
    """None when got equals want bit for bit (NaN by position), else a description of where they differ."""
    gn, wn = np.isnan(got), np.isnan(want)
    bad = ((got.view(np.uint32) != want.view(np.uint32)) & ~(gn & wn)).any(axis=-1)
    if not bad.any():
        return None
    ys, xs = np.nonzero(bad)
    first = [dict(x=int(x), y=int(y), x_mod64=int(x % 64), x_mod4=int(x % 4), y_mod32=int(y % 32), y_mod16=int(y % 16),
                  got=got[y, x].tolist(), want=want[y, x].tolist()) for y, x in zip(ys[:n], xs[:n])]
    return dict(pixels=int(bad.sum()), of=int(bad.size), first=first)


def _check_exact(got, want, label, fails):
    m = _mismatch(got, want)
    print(f"{label}: {'bit-identical' if m is None else str(m['pixels']) + ' pixels differ'}")
    if m is not None:
        fails.append((label, m))


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


def _model(I0, I1, P, init=None, kernel_path=0):
    return fn.calc(I0, I1, P, init_flow=init, build="eng", order=fn.order_for(P, kernel_path))


def _grid(n, rx=29, ry=17):
    """rows, cols of a level with n 64 x 32 tiles (tx * ty == n) and ragged right and bottom edges."""
    tx = max(d for d in range(1, int(n ** 0.5) + 1) if n % d == 0)
    ty = n // tx
    return (ty - 1) * FT_H + ry, (tx - 1) * FT_W + rx


def _sweep_shapes(n_sm):
    """(rows, cols, why, flags): the box window at the tile counts around the 512-thread kernel's limit, both windows
    at every column residue, rows at and across the running sum's 16-row strip starts past n_SM tiles, then small
    shapes with the two windows alternating."""
    shapes = [(*_grid(n), f"{n} tiles", 0) for n in (n_sm, n_sm + 1, 2 * n_sm + 1)]
    ty = 12
    tx = -(-(2 * n_sm + 1) // ty)  # at least 2 n_SM + 1 tiles
    shapes += [((ty - 1) * FT_H + 12, (tx - 1) * FT_W + r, f"cols % 4 == {((tx - 1) * FT_W + r) % 4}, {tx * ty} tiles",
                flags) for r in (29, 30, 31, 32) for flags in (0, 256)]
    wide = 64 * (n_sm + 1) + 13   # one tile row of more than n_SM tiles: the 256-thread kernels
    shapes += [(r, wide, "strip edge", 0) for r in (15, 16, 17, 47, 48, 49)]
    small = [(r, 301, "vertical window") for r in (WIN - 1, WIN, WIN + 1, FT_H - 1)]
    small += [(1, 37, "1xN"), (37, 1, "Nx1"), (2, 2, "2x2"), (3, 5, "3x5")]
    return shapes + [(h, w, why, 256 * (i % 2)) for i, (h, w, why) in enumerate(small)]


def _sweep_case(i, flags):
    kw = dict(ONE_LEVEL, flags=flags, **(dict(polyN=7, polySigma=1.5) if i % 4 >= 2 else {}))
    return kw, ("f32" if i % 3 == 1 else "u8")


def test_shape_sweep_vs_model(cuda_device, stream, num_sms):
    """One level, default kernel, box / gaussian, polyN 5 / 7 and u8 / f32 input alternating; the round-1 blur and
    polynomial-expansion kernels (aux_path 6) give the same bits."""
    t0, fails = time.time(), []
    for i, (h, w, why, flags) in enumerate(_sweep_shapes(num_sms)):
        kw, dtype = _sweep_case(i, flags)
        I0, I1 = _pair(h, w, seed=40 + i, dtype=dtype)
        got, alg = _engine(cuda_device, stream, I0, I1, **kw)
        P = _params(kw)
        paths = _check_paths(alg, h, w, P, num_sms)
        label = f"sweep {h}x{w} {dtype} {kw} ({why}) {paths}"
        _check_exact(got, _model(I0, I1, P), label, fails)
        r1, _ = _engine(cuda_device, stream, I0, I1, aux_path=6, **kw)
        _check_exact(r1, got, label + " aux_path 6 vs default", fails)
    print(f"sweep: {time.time() - t0:.1f} s")
    assert not fails, fails


def test_iteration_kernel_variants_vs_model(cuda_device, stream, num_sms):
    """kernel_path 0 / 1 / 2 and aux_path 3 / 4 / 5 at a level past n_SM tiles, box and gaussian, on one handle (each
    change of knob re-captures the graph; the repeat call replays it and must report the same kernels).  Each equals the
    model in its own iteration order: kernel_path 1 (k_farn_iter) sums the box window pair by pair and rounds the first
    gaussian tap on its own, the others run the K = 6 order."""
    h, w = _grid(2 * num_sms + 1)
    fails = []
    for flags in (0, 256):
        kw = dict(ONE_LEVEL, flags=flags)
        P = _params(kw)
        I0, I1 = _pair(h, w, seed=7 + flags, dtype="u8")
        want = {o: _model(I0, I1, P, kernel_path=1 if o == "generic" else 0) for o in ("fast", "generic")}
        assert _mismatch(want["fast"], want["generic"]) is not None   # the two orders round differently
        alg = None
        for kp, aux in ((0, 0), (1, 0), (2, 0), (0, 3), (0, 4), (0, 5)):
            got, alg = _engine(cuda_device, stream, I0, I1, kernel_path=kp, aux_path=aux, alg=alg, **kw)
            paths = _check_paths(alg, h, w, P, num_sms, kernel_path=kp, aux_path=aux)
            again, _ = _engine(cuda_device, stream, I0, I1, kernel_path=kp, aux_path=aux, alg=alg, **kw)
            assert np.array_equal(again, got) and _check_paths(alg, h, w, P, num_sms, kernel_path=kp,
                                                               aux_path=aux) == paths
            _check_exact(got, want[fn.order_for(P, kp)], f"{h}x{w} flags {flags} kernel_path {kp} aux_path {aux} {paths}",
                         fails)
    assert not fails, fails


def test_persistent_tma_kernel_vs_model(cuda_device, stream, num_sms):
    """kernel_path 3 on levels with at least 2 n_SM + 1 64 x 64 tiles, ragged in both directions, at every column residue
    mod 4 (must run the TMA kernel and equal the model), and on a level just below the threshold (must report the fast
    kernel and equal the model)."""
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
        _check_exact(got, _model(I0, I1, P, kernel_path=3), f"tma {h}x{w} cols % 4 == {w % 4} {paths}", fails)
    tx = (2 * num_sms - 1) // ty   # tx * ty < 2 n_SM
    h, w = (ty - 1) * TT + 23, (tx - 1) * TT + 29
    I0, I1 = _pair(h, w, seed=70, dtype="u8")
    got, alg = _engine(cuda_device, stream, I0, I1, kernel_path=3, **ONE_LEVEL)
    paths = _check_paths(alg, h, w, _params(ONE_LEVEL), num_sms, kernel_path=3)
    assert FARN_PATH["tma"] not in paths
    _check_exact(got, _model(I0, I1, _params(ONE_LEVEL), kernel_path=3), f"tma below threshold {h}x{w} {paths}", fails)
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
        _check_exact(got, _model(I0, I1, P), f"winSize {win} flags {flags} {paths}", fails)
    assert not fails, fails


# (name, create() arguments): each stage adds one part of the pipeline to the one before
LADDER = [
    ("1 level, 1 iteration", dict(numLevels=0, numIters=1)),
    ("1 level, 2 iterations", dict(numLevels=0, numIters=2)),
    ("2 levels", dict(numLevels=1, numIters=2)),
    ("fastPyramids", dict(numLevels=2, numIters=2, fastPyramids=True)),
    ("initial flow", dict(numLevels=2, numIters=2, flags=fm.OPTFLOW_USE_INITIAL_FLOW)),
    ("gaussian", dict(numLevels=2, numIters=2, flags=fm.OPTFLOW_FARNEBACK_GAUSSIAN)),
]


def test_stage_ladder_vs_model(cuda_device, stream, num_sms):
    """The pipeline stage by stage at a level past n_SM tiles; the first stage that differs is named."""
    h, w = _grid(n_sm_tiles := num_sms + 3, rx=45, ry=27)
    I0, I1 = _pair(h, w, seed=90, dtype="u8")
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    init = np.stack([2.5 * np.sin(xx / 37.0), 1.5 * np.cos(yy / 23.0)], axis=-1).astype(np.float32)
    for name, kw in LADDER:
        P = _params(kw)
        ini = init if kw.get("flags", 0) & fm.OPTFLOW_USE_INITIAL_FLOW else None
        got, alg = _engine(cuda_device, stream, I0, I1, init=ini, **kw)
        paths = _check_paths(alg, h, w, P, num_sms)
        m = _mismatch(got, _model(I0, I1, P, ini))
        print(f"ladder {name} ({h}x{w}, {n_sm_tiles} tiles) {paths}: {'bit-identical' if m is None else m['pixels']}")
        assert m is None, f"first stage that differs: {name}: {m}"


@pytest.mark.parametrize("pyr_scale,h,w", [(0.7, 211, 307), (0.7, 150, 401), (0.5, 211, 307)])
def test_pyramid_scales_vs_model(cuda_device, stream, num_sms, pyr_scale, h, w):
    """pyrScale 0.7 at odd sizes (non-integral 1 / scale: both bilinear rows of the level image, ystep 1) and 0.5
    (integral: odd staging rows not launched, ystep 2), box and gaussian."""
    fails = []
    for flags in (0, 256):
        kw = dict(numLevels=3, numIters=3, pyrScale=pyr_scale, flags=flags)
        P = _params(kw)
        I0, I1 = _pair(h, w, seed=100 + h, dtype="u8")
        got, alg = _engine(cuda_device, stream, I0, I1, **kw)
        paths = _check_paths(alg, h, w, P, num_sms)
        _check_exact(got, _model(I0, I1, P), f"pyrScale {pyr_scale} {h}x{w} flags {flags} {paths}", fails)
    assert not fails, fails


@pytest.mark.parametrize("mag", [1e4, 3e38])
def test_wild_initial_flow_vs_model(cuda_device, stream, num_sms, mag):
    """An initial flow pointing far outside the image (the floor clamp of updateMatrices); NaN by position."""
    h, w = 97, 203
    I0, I1 = _pair(h, w, seed=110, dtype="u8")
    rng = np.random.default_rng(5)
    init = (rng.choice([-1.0, 1.0, 0.25], size=(h, w, 2)) * mag).astype(np.float32)
    kw = dict(numLevels=0, numIters=2, flags=fm.OPTFLOW_USE_INITIAL_FLOW)
    P = _params(kw)
    got, alg = _engine(cuda_device, stream, I0, I1, init=init, **kw)
    _check_paths(alg, h, w, P, num_sms)
    m = _mismatch(got, _model(I0, I1, P, init))
    assert m is None, m


def test_constant_frames_vs_model(cuda_device, stream, num_sms):
    """Constant frames: every polynomial coefficient but the constant one is zero and the 2x2 systems are singular up
    to the 1e-3 regulariser."""
    fails = []
    for kw in (dict(numLevels=2, numIters=3), dict(numLevels=2, numIters=3, flags=256)):
        I0 = np.full((120, 250), 77, np.uint8)
        I1 = np.full((120, 250), 78, np.uint8)
        got, alg = _engine(cuda_device, stream, I0, I1, **kw)
        _check_paths(alg, 120, 250, _params(kw), num_sms)
        _check_exact(got, _model(I0, I1, _params(kw)), f"constant {kw}", fails)
    assert not fails, fails


def test_pitched_roi_vs_model(cuda_device, stream):
    """u8 and f32 inputs that are views into larger images (row pitch != width), and an initial flow / result that is a
    view into a larger flow field: the same bits as the model of the cropped data, and nothing outside the view
    written."""
    import torch
    import opencv_contrib_b200 as ocb
    h, w, H, W = 133, 251, 150, 300
    fails = []
    for dtype in ("u8", "f32"):
        B0, B1 = _pair(H, W, seed=120, dtype=dtype)
        I0, I1 = B0[9:9 + h, 21:21 + w], B1[9:9 + h, 21:21 + w]
        yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
        big = np.stack([np.sin(xx / 29.0), np.cos(yy / 31.0)], axis=-1).astype(np.float32)
        kw = dict(numLevels=2, numIters=3, flags=fm.OPTFLOW_USE_INITIAL_FLOW)
        alg = ocb.FarnebackOpticalFlow_create(**kw)
        d0 = torch.from_numpy(B0).to(cuda_device)[9:9 + h, 21:21 + w]
        d1 = torch.from_numpy(B1).to(cuda_device)[9:9 + h, 21:21 + w]
        fbig = torch.from_numpy(big).to(cuda_device)
        fl = fbig[5:5 + h, 11:11 + w]
        assert fl.stride(0) == 2 * W and d0.stride(0) == W
        alg.calc(d0, d1, fl, stream)
        stream.synchronize()
        out = fbig.cpu().numpy()
        want = _model(np.ascontiguousarray(I0), np.ascontiguousarray(I1), _params(kw),
                      np.ascontiguousarray(big[5:5 + h, 11:11 + w]))
        _check_exact(out[5:5 + h, 11:11 + w], want, f"ROI {dtype}", fails)
        outside = np.ones((H, W), bool)
        outside[5:5 + h, 11:11 + w] = False
        assert np.array_equal(out[outside], big[outside]), dtype
    assert not fails, fails


_BENCH_MODELS = {}


def _bench_case(name):
    """Input, parameters and model result of one 1080p case, computed once per module."""
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
        ref = _model(I0, I1, _params(kw), init)
        print(f"1080p {name}: model {time.time() - t0:.1f} s")
        _BENCH_MODELS[name] = (I0, I1, kw, init, ref)
    return _BENCH_MODELS[name]


@pytest.mark.parametrize("name,kernel_path", [("default", 0), ("default", 3), ("gaussian", 0), ("fastPyramids", 0),
                                              ("initial_flow", 0)])
def test_benchmark_size_vs_model(cuda_device, stream, num_sms, name, kernel_path):
    """1080p with the benchmark's parameters (5 levels, winSize 13, 10 iterations, polyN 5, f32 input); the default
    case also through the round-1 blur and polynomial-expansion kernels (aux_path 6)."""
    I0, I1, kw, init, ref = _bench_case(name)
    h, w = I0.shape
    got, alg = _engine(cuda_device, stream, I0, I1, kernel_path=kernel_path, init=init, **kw)
    assert alg.getStats()["levels"] == len(fm.level_sizes(h, w, _params(kw))) == 6
    paths = _check_paths(alg, h, w, _params(kw), num_sms, kernel_path=kernel_path)
    fails = []
    _check_exact(got, ref, f"1080p {name} kernel_path {kernel_path} {paths}", fails)
    if name == "default" and kernel_path == 0:
        r1, _ = _engine(cuda_device, stream, I0, I1, aux_path=6, **kw)
        _check_exact(r1, got, "1080p aux_path 6 vs default", fails)
    assert not fails, fails
