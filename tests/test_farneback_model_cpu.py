"""The Farneback CUDA-semantics models: the numpy model's precision parameter (oracle/farneback_gpu_model.py,
calc(precision=...)) and its C restatement (oracle/farneback_model.c).

* precision "f32": its flows must stay bit for bit what the float-only model computed before the parameter existed
  (tests/golden/farneback_model_f32_digests.json holds SHA-256 digests of those flows, recorded with that model), and the
  C build "f32" must equal it bit for bit;
* the C build "eng" carries the engine's roundings (the model the GPU tests compare with exactly): each of its
  departures from "f32" must matter on its own, it must stay within rounding distance of "f32", and its running box
  sum must match a direct restatement;
* precision "f64" is the yardstick of that rounding distance: it must run at every edge shape the GPU sweep uses and
  stay close to "f32" there;
* the f32-vs-f64 distance at the GPU test configurations is printed, so a run records it.
"""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import metrics, synth, farneback_gpu_model as fm

GOLD = os.path.join(os.path.dirname(__file__), "golden", "farneback_model_f32_digests.json")

# (rows, cols, seed, input type, create() arguments, initial flow)
DIGEST_CASES = [
    (72, 96, 1, "u8", dict(), False),
    (72, 96, 2, "u8", dict(flags=256), False),
    (72, 96, 3, "u8", dict(polyN=7, polySigma=1.5), False),
    (72, 96, 4, "u8", dict(fastPyramids=True), False),
    (81, 101, 5, "u8", dict(pyrScale=0.8, numLevels=3), False),
    (72, 96, 6, "f32", dict(winSize=9, flags=256), False),
    (27, 90, 7, "u8", dict(numLevels=0, numIters=3, winSize=1), False),
    (1, 37, 8, "u8", dict(numLevels=0, numIters=3), False),
    (37, 1, 9, "u8", dict(numLevels=0, numIters=3, flags=256), False),
    (2, 2, 10, "u8", dict(numLevels=0, numIters=3), False),
    (72, 96, 11, "u8", dict(flags=4), True),
]


def _pair(h, w, seed, dtype):
    I0, I1, gt = synth.make_pair(max(h, 16), max(w, 16), seed=seed, kind="smooth", dtype="f32" if dtype == "f32" else "u8")
    if dtype == "f32":
        I0, I1 = I0 * np.float32(255), I1 * np.float32(255)
    return np.ascontiguousarray(I0[:h, :w]), np.ascontiguousarray(I1[:h, :w]), np.ascontiguousarray(gt[:h, :w])


def _case_flow(h, w, seed, dtype, kw, use_init, precision="f32"):
    I0, I1, gt = _pair(h, w, seed, dtype)
    init = (gt + 0.3).astype(np.float32) if use_init else None
    return fm.calc(I0, I1, fm.FarnebackParams(**kw), init_flow=init, precision=precision)


def test_f32_model_bit_identical_to_recorded_flows():
    want = json.load(open(GOLD))
    assert len(want) == len(DIGEST_CASES)
    for case, digest in zip(DIGEST_CASES, want):
        f = _case_flow(*case)
        assert f.dtype == np.float32
        assert hashlib.sha256(np.ascontiguousarray(f).tobytes()).hexdigest() == digest, case


@pytest.mark.parametrize("h,w,kw", [
    (1, 37, dict()), (37, 1, dict()), (2, 2, dict()), (3, 5, dict(flags=256)),
    (20, 70, dict()), (27, 301, dict(flags=256)), (31, 301, dict(polyN=7, polySigma=1.5)),
    (60, 80, dict(winSize=1)), (60, 80, dict(winSize=1, flags=256))])
def test_f64_model_at_edge_shapes(h, w, kw):
    """One level, 3 iterations (the GPU sweep's settings): f64 runs in double throughout and stays near f32."""
    kw = dict(numLevels=0, numIters=3, **kw)
    I0, I1, _ = _pair(h, w, 30, "u8")
    P = fm.FarnebackParams(**kw)
    stages = {}
    f64 = fm.calc(I0, I1, P, precision="f64", stages=stages)
    f32 = fm.calc(I0, I1, P)
    assert f64.dtype == np.float64 and stages["R"][(0, 0)].dtype == np.float64 and stages["M0"][0].dtype == np.float64
    assert np.isfinite(f64).all() and f64.shape == (h, w, 2)
    e = metrics.epe(f32, f64)
    # winSize 1 solves every pixel from its own 2x2 system: where it is near singular 1 / (det + 1e-3) amplifies
    # rounding far beyond the window-averaged sizes, so only the median is bounded tightly there
    print(f"{h}x{w} {kw}: f32-vs-f64 q50 {np.quantile(e, 0.5):.2e} q99 {np.quantile(e, 0.99):.2e} max {e.max():.2e}")
    assert np.quantile(e, 0.5) <= 5e-5
    if kw.get("winSize", 13) > 1:
        assert e.max() <= 1e-3


def test_f32_vs_f64_distance_at_gpu_configurations():
    """Records the yardstick at small versions of the GPU test configurations (full-size figures: DESIGN.md)."""
    for h, w, kw in [(240, 320, dict()), (240, 320, dict(flags=256)), (240, 320, dict(fastPyramids=True)),
                     (240, 320, dict(polyN=7, polySigma=1.5)), (300, 700, dict(numLevels=0, numIters=3, winSize=31)),
                     (364, 1439, dict(numLevels=0, numIters=3))]:
        I0, I1, _ = _pair(h, w, 3, "u8")
        P = fm.FarnebackParams(**kw)
        e = metrics.epe(fm.calc(I0, I1, P), fm.calc(I0, I1, P, precision="f64"))
        qs = [float(np.quantile(e, q)) for q in (0.5, 0.99, 0.999, 1.0)]
        print(f"{h}x{w} {kw}: f32-vs-f64 q50 {qs[0]:.2e} q99 {qs[1]:.2e} q99.9 {qs[2]:.2e} max {qs[3]:.2e}")
        assert np.isfinite(e).all() and qs[0] <= 1e-5 and qs[1] <= 1e-3


# ---- the C restatement, oracle/farneback_model.c (farneback_model_native) ----

from oracle import farneback_model_native as fn  # noqa: E402


def _case_inputs(h, w, seed, dtype, kw, use_init):
    I0, I1, gt = _pair(h, w, seed, dtype)
    return I0, I1, fm.FarnebackParams(**kw), ((gt + 0.3).astype(np.float32) if use_init else None)


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def test_c_f32_model_bit_identical_to_numpy_model():
    """The C f32 build restates calc(precision="f32") operation for operation, so the recorded digests pin it too."""
    want = json.load(open(GOLD))
    for case, digest in zip(DIGEST_CASES, want):
        I0, I1, P, init = _case_inputs(*case)
        got = fn.calc(I0, I1, P, init_flow=init, build="f32")
        assert _same_bits(got, fm.calc(I0, I1, P, init_flow=init)), case
        assert hashlib.sha256(got.tobytes()).hexdigest() == digest, case


@pytest.mark.parametrize("switch", fn.SWITCHES)
def test_each_engine_rounding_switch_is_live(switch):
    """Each departure of the engine model from f32, switched on alone, changes the result.  The floor clamp is the
    exception: a displacement it clamps has no bilinear cell either way, so it must leave every bit alone, even for
    flows far outside the image."""
    build = "only_" + switch
    assert fn.lib(build).farneback_model_switches() == 1 << fn.SWITCHES.index(switch)
    if switch == "SKIP_ZERO":
        # a zero-weight tap on an infinite sample adds inf * 0 = NaN unless it is skipped
        src = np.full((40, 60), 10, np.float32)
        src[::2, 7] = np.inf
        taps = fm.gaussian_kernel_half(3, 0.5)
        a, b = (fn.level_image(src, taps, 20, 30, build=x) for x in ("f32", build))
        assert np.isnan(a).any() and not _same_bits(a, b)
        return
    I0, I1, _ = _pair(72, 96, 3, "f32")   # non-integral values: pyr_tap5 and cv2.pyrDown round apart
    kw = dict(numLevels=2, numIters=3)
    init = None
    if switch == "PYR_TAP5":
        kw["fastPyramids"] = True
    elif switch in ("FUSED_RESIZE", "FLOOR_CLAMP"):
        kw["pyrScale"] = 0.7   # bilinear weights that are not powers of two
        kw["flags"] = fm.OPTFLOW_USE_INITIAL_FLOW
        yy, xx = np.mgrid[0:72, 0:96].astype(np.float32)
        init = np.stack([np.sin(xx / 7.0), np.cos(yy / 5.0)], -1).astype(np.float32)
        if switch == "FLOOR_CLAMP":
            init = init * np.float32(3e38)
            kw["numLevels"] = 0
    P = fm.FarnebackParams(**kw)
    a = fn.calc(I0, I1, P, init_flow=init, build="f32")
    b = fn.calc(I0, I1, P, init_flow=init, build=build)
    both_nan = np.isnan(a) & np.isnan(b)
    same = bool(((a.view(np.uint32) == b.view(np.uint32)) | both_nan).all())
    assert same if switch == "FLOOR_CLAMP" else not same


def _running_box_numpy(P):
    """The box window of k_farn_iter_fast restated directly: per 16-row strip a balanced tree over the 13 rows around its
    first row, then acc + (new - old); per 4-pixel task the same across columns; replicate border; times 1/169."""
    F = np.float32
    h, w = P.shape

    def tree(v):
        a = (v[0] + v[1]) + (v[2] + v[3])
        b = (v[4] + v[5]) + (v[6] + v[7])
        c = (v[8] + v[9]) + (v[10] + v[11])
        return ((a + b) + c) + v[12]

    V = np.empty_like(P)
    for y0 in range(0, h, 16):
        v = [P[min(max(y0 - 6 + q, 0), h - 1)] for q in range(28)]
        acc = tree(v)
        for o in range(min(16, h - y0)):
            if o:
                acc = acc + (v[o + 12] - v[o - 1])
            V[y0 + o] = acc
    out = np.empty_like(P)
    for x0 in range(0, w, 4):
        c = [V[:, min(max(x0 - 6 + q, 0), w - 1)] for q in range(16)]
        acc = tree(c)
        for e in range(min(4, w - x0)):
            if e:
                acc = acc + (c[e + 12] - c[e - 1])
            out[:, x0 + e] = acc * F(1.0 / 169)
    return out


def test_running_box_sum_matches_direct_restatement():
    rng = np.random.default_rng(3)
    M = rng.standard_normal((5, 53, 71)).astype(np.float32) * np.float32(100)
    got = fn.box(M, 13, order="fast", build="eng")
    for p in range(5):
        assert _same_bits(got[p], _running_box_numpy(M[p])), p
    # the generic order is the numpy model's pair-by-pair sum, and the two orders differ
    assert _same_bits(fn.box(M, 13, order="generic", build="eng"), fm.box_filter5(M, 6))
    assert not _same_bits(got, fm.box_filter5(M, 6))


def test_engine_model_within_float_rounding_of_f32_model():
    """eng departs from f32 by rounding alone: at every quantile its end-point error against f32 stays within 4 x the
    f32-vs-f64 error of the same input (the tolerance the GPU tests used to apply).  No code path of either model
    depends on the frame size beyond the level count and the border cases these sizes already reach, so 1080p (where
    the numpy double model takes minutes) is not repeated here."""
    for h, w, kw in [(240, 320, dict()), (240, 320, dict(flags=256)), (240, 320, dict(fastPyramids=True)),
                     (240, 320, dict(flags=fm.OPTFLOW_USE_INITIAL_FLOW)), (364, 1439, dict(numLevels=0, numIters=3))]:
        I0, I1, gt = _pair(h, w, 3, "u8")
        init = (gt + 0.3).astype(np.float32) if kw.get("flags", 0) & fm.OPTFLOW_USE_INITIAL_FLOW else None
        P = fm.FarnebackParams(**kw)
        f32 = fm.calc(I0, I1, P, init_flow=init)
        yard = metrics.epe(f32, fm.calc(I0, I1, P, init_flow=init, precision="f64"))
        e = metrics.epe(fn.calc(I0, I1, P, init_flow=init, build="eng", order=fn.order_for(P)), f32)
        for q in (0.5, 0.99, 0.999, 1.0):
            v, y = float(np.quantile(e, q)), float(np.quantile(yard, q))
            assert v <= 4 * y, (h, w, kw, q, v, y)


def test_engine_model_thread_count_invariant():
    I0, I1, _ = _pair(150, 230, 9, "u8")
    P = fm.FarnebackParams(numLevels=2, numIters=3)
    try:
        fn.set_threads(1)
        one = fn.calc(I0, I1, P, build="eng")
        fn.set_threads(8)
        eight = fn.calc(I0, I1, P, build="eng")
    finally:
        from oracle.tvl1_cpu_native import usable_cpus
        fn.set_threads(usable_cpus())
    assert _same_bits(one, eight)


def test_engine_model_time_at_1080p():
    """The engine model at the benchmark's parameters (1080p, 5 levels, winSize 13, 10 iterations): prints its time."""
    import time
    I0, I1, _ = synth.make_pair(1080, 1920, seed=0, kind="smooth", dtype="f32")
    t0 = time.time()
    f = fn.calc(I0 * np.float32(255), I1 * np.float32(255), fm.FarnebackParams(), build="eng")
    print(f"eng model, 1080p bench parameters: {time.time() - t0:.2f} s on {fn.set_threads(0)} threads")
    assert np.isfinite(f).all()
