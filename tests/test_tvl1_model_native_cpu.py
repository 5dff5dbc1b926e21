"""CPU tests of oracle/tvl1_gpu_model.c, the native restatement of the CUDA-semantics model that the full-size GPU
tests (tests/test_tvl1_fullsize_gpu.py) compare the engine with.

  * The float build equals the numpy model (oracle/tvl1_gpu_model.py) bit for bit, iteration traces included.  The
    libm calls both make -- floorf / ceilf (exact) and hypotf in the dual update (numpy's float32 hypot is libm's
    hypotf) -- do not break bit-equality: the flows below compare as raw bits.
  * The error image is summed in numpy's pairwise order, so the epsilon cadence decides as the numpy model does.
  * The double build is the yardstick for float rounding; its distance from the float build at the GPU tests'
    small-size configurations is recorded here, and it is what allows the 1e-3 px bound there.
"""
import numpy as np
import pytest

from oracle import metrics, synth, tvl1_gpu_model as gm, tvl1_gpu_model_native as nm


@pytest.fixture(scope="module", autouse=True)
def _built():
    if not (nm.available("f32") and nm.available("f64")):
        import __graft_entry__ as g
        g.build()


def _pair(h, w, seed, dtype="u8", kind="smooth"):
    I0, I1, gt = synth.make_pair(max(h, 16), max(w, 16), seed=seed, kind=kind, dtype=dtype)
    return np.ascontiguousarray(I0[:h, :w]), np.ascontiguousarray(I1[:h, :w])


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _same(I0, I1, init=None, **kw):
    P = gm.TVL1Params(**kw)
    ta, tb = [], []
    a = gm.calc(I0, I1, P, init_flow=init, trace=ta)
    b = nm.calc(I0, I1, P, init_flow=init, trace=tb)
    assert b.dtype == np.float32 and _bits_equal(a, b), float(np.abs(a.astype(np.float64) - b).max())
    assert ta == tb
    return ta


SMALL = dict(nscales=4, warps=3, epsilon=0.0, iterations=20)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 37), (37, 1), (17, 23), (97, 131), (243, 317)])
@pytest.mark.parametrize("dtype", ["u8", "f32"])
def test_float_build_bit_identical_to_numpy_model(h, w, dtype):
    I0, I1 = _pair(h, w, seed=h + w, dtype=dtype)
    _same(I0, I1, **SMALL)


def test_gamma_and_scale_step():
    I0, I1 = _pair(97, 131, seed=3, dtype="f32")
    _same(I0, I1, nscales=3, warps=2, epsilon=0.0, iterations=10, gamma=1.0)
    _same(I0, I1, nscales=4, warps=2, epsilon=0.0, iterations=10, scaleStep=0.5)
    _same(I0, I1, nscales=3, warps=2, epsilon=0.0, iterations=10, scaleStep=0.65)


@pytest.mark.parametrize("amp", [0.7, 11.5, 40.0])
def test_initial_flow_pointing_out_of_the_image(amp):
    h, w = 97, 131
    I0, I1 = _pair(h, w, seed=5)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    # left / up in the left / top half, right / down in the other: a good part of the warped taps lands outside
    init = np.stack([amp * np.sign(xx - w / 2) + np.sin(yy / 7.0), amp * np.sign(yy - h / 2) + np.cos(xx / 5.0)],
                    axis=-1).astype(np.float32)
    _same(I0, I1, init=init, nscales=3, warps=2, epsilon=0.0, iterations=10, useInitialFlow=True)


def test_early_stop_below_16_pixels():
    I0, I1 = _pair(40, 40, seed=6)
    assert gm.level_sizes(40, 40, 8, 0.5)[1] == 2
    assert len(_same(I0, I1, nscales=8, warps=2, epsilon=0.0, iterations=10, scaleStep=0.5)) == 2
    I0, I1 = _pair(20, 300, seed=7)
    assert len(_same(I0, I1, nscales=5, warps=2, epsilon=0.0, iterations=10)) == 2  # rows stop it


@pytest.mark.parametrize("kw", [dict(nscales=3, warps=3, epsilon=0.01, iterations=100),
                                dict(nscales=2, warps=2, epsilon=0.05, iterations=37),
                                dict()])  # the reference's create() defaults
def test_epsilon_cadence_traces_match(kw):
    I0, I1 = _pair(120, 160, seed=2, kind="const")
    trace = _same(I0, I1, **kw)
    counts = [n for level in trace for n in level]
    assert any(n < (kw.get("iterations", 300)) for n in counts)  # the stopping rule did end some warps early


def test_error_sum_is_numpys_pairwise_sum():
    a = (np.random.default_rng(0).random(1_000_003).astype(np.float32) ** 2) * np.float32(3e-3)
    for n in (1, 7, 8, 9, 127, 128, 129, 1000, 65537, 1_000_003):
        assert nm.error_sum(a[:n]) == float(a[:n].astype(np.float64).sum()), n


def test_double_build_yardstick_at_small_gpu_test_configs():
    """Float vs double at the inputs of tests/test_tvl1_gpu.py's model comparisons (4 scales x 3 warps x 20
    iterations).  Measured: max 1.5e-4 / 9.5e-5 / 4.1e-5 px; the engine's 1e-3 bound there is >= 4x these."""
    for (h, w, kind, seed), measured in (((120, 160, "const", 0), 1.5e-4), ((243, 317, "smooth", 1), 9.5e-5),
                                         ((97, 131, "affine", 2), 4.1e-5)):
        I0, I1, _ = synth.make_pair(h, w, seed=seed, kind=kind)
        P = gm.TVL1Params(**SMALL)
        a, b = nm.calc(I0, I1, P), nm.calc(I0, I1, P, precision="f64")
        assert b.dtype == np.float64
        e = metrics.epe(a, b)
        assert 0 < e.max() <= 2 * measured and 4 * e.max() <= 1e-3, (h, w, e.max())
