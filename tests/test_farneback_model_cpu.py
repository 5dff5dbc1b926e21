"""The Farneback CUDA-semantics model's precision parameter (oracle/farneback_gpu_model.py, calc(precision=...)).

* precision "f32" is the model every Farneback GPU test compares against: its flows must stay bit for bit what the
  float-only model computed before the parameter existed (tests/golden/farneback_model_f32_digests.json holds SHA-256
  digests of those flows, recorded with that model);
* precision "f64" is the yardstick of tests/test_farneback_fullsize_gpu.py: it must run at every edge shape the GPU
  sweep uses and stay close to "f32" there;
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
