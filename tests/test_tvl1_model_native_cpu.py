"""CPU tests of oracle/tvl1_gpu_model.c, the native restatement of the CUDA-semantics model that the full-size GPU
tests (tests/test_tvl1_fullsize_gpu.py) compare the engine with.

  * The float build equals the numpy model (oracle/tvl1_gpu_model.py) bit for bit, iteration traces included.  The
    libm calls both make -- floorf / ceilf (exact) and hypotf in the dual update (numpy's float32 hypot is libm's
    hypotf) -- do not break bit-equality: the flows below compare as raw bits.
  * The error image is summed in numpy's pairwise order, so the epsilon cadence decides as the numpy model does.
  * The double build is the yardstick for float rounding; its distance from the float build at the GPU tests'
    small-size configurations is recorded here.
  * The engine-rounding build ("eng", the model the engine must equal bit for bit): its emulation of rcp.approx /
    sqrt.approx, fed tables of the correctly rounded operations, is 1/x and sqrt(x) wherever the result is normal and
    flushes as .ftz says; fed those tables it stays within FACTOR x (float vs double) of the float build, so the
    engine's departures cannot grow into an error the float yardstick would not allow; and no build's result depends
    on the OpenMP thread count.  (The device tables, and the emulation against the device on all 2^32 inputs, are
    tests/test_tvl1_gpu.py's.)
"""
import numpy as np
import pytest

from oracle import metrics, mufu, synth, tvl1_gpu_model as gm, tvl1_gpu_model_native as nm

FACTOR = 4.0  # as in tests/test_tvl1_fullsize_gpu.py


@pytest.fixture(scope="module", autouse=True)
def _built():
    if not (nm.available("f32") and nm.available("f64") and nm.available("eng")):
        import __graft_entry__ as g
        g.build()


@pytest.fixture(scope="module")
def eng_cr():
    """The "eng" build fed the correctly rounded tables."""
    nm.set_mufu_tables(*mufu.correctly_rounded_tables())
    return nm


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


def test_mufu_emulation_on_correctly_rounded_tables(eng_cr):
    import torch
    x = mufu.sample_inputs()
    with np.errstate(invalid="ignore"):
        x64 = x.astype(np.float64)
    bits = x.view(np.uint32)
    e = (bits >> 23) & 0xFF
    neg = (bits >> 31) == 1
    normal_in = (e > 0) & (e < 255)
    tabs = [torch.from_numpy(t.view(np.int32)) for t in mufu.correctly_rounded_tables()]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ieee = {mufu.OP_RCP: (1.0 / x64).astype(np.float32), mufu.OP_SQRT: np.sqrt(x64).astype(np.float32)}
    for op in (mufu.OP_RCP, mufu.OP_SQRT):
        got = eng_cr.mufu_apply(op, x)
        # the C emulation and the torch statement of the rule (what the GPU test checks on the device) agree
        pred = mufu.predict(op, torch.from_numpy(x.view(np.int32)), *tabs).numpy().view(np.float32)
        same = (got.view(np.uint32) == pred.view(np.uint32)) | (np.isnan(got) & np.isnan(pred))
        assert same.all(), (op, x[~same][:8])
        ref = ieee[op]
        ok = normal_in & (np.abs(ref) >= np.finfo(np.float32).tiny) & np.isfinite(ref)
        assert ok.sum() > 1_000_000
        assert np.array_equal(got[ok].view(np.uint32), ref[ok].view(np.uint32)), op
        zero_in = e == 0
        if op == mufu.OP_RCP:
            assert np.array_equal(got[zero_in], np.where(neg[zero_in], -np.inf, np.inf).astype(np.float32))
            flushed = normal_in & (np.abs(ref) < np.finfo(np.float32).tiny)
            assert flushed.sum() > 0 and np.all(got[flushed] == 0)
            assert np.array_equal(np.signbit(got[flushed]), neg[flushed])
            inf_in = np.isinf(x)
            assert np.all(got[inf_in] == 0) and np.array_equal(np.signbit(got[inf_in]), neg[inf_in])
        else:
            assert np.all(got[zero_in] == 0) and np.array_equal(np.signbit(got[zero_in]), neg[zero_in])
            assert np.isnan(got[neg & ~zero_in]).all()
            assert np.isposinf(got[np.isposinf(x)]).all()
        assert np.isnan(got[np.isnan(x)]).all()


@pytest.mark.parametrize("case", ["const", "smooth", "affine", "gamma"])
def test_engine_rounding_build_within_float_yardstick(eng_cr, case):
    """With correctly rounded tables, the engine's roundings move the flow no further from the float model than
    FACTOR x the float model's own distance from the double model, at the small GPU-test configurations."""
    (h, w, kind, seed), kw = {"const": ((120, 160, "const", 0), SMALL), "smooth": ((243, 317, "smooth", 1), SMALL),
                              "affine": ((97, 131, "affine", 2), SMALL),
                              "gamma": ((120, 160, "const", 2), dict(nscales=3, warps=3, epsilon=0.0, iterations=20,
                                                                     gamma=1.0))}[case]
    I0, I1, _ = synth.make_pair(h, w, seed=seed, kind=kind)
    P = gm.TVL1Params(**kw)
    f32 = nm.calc(I0, I1, P)
    yard = metrics.epe(f32, nm.calc(I0, I1, P, precision="f64"))
    e = metrics.epe(nm.calc(I0, I1, P, precision="eng"), f32)
    for q in (0.5, 0.99, 1.0):
        v, y = float(np.quantile(e, q)), float(np.quantile(yard, q))
        assert v <= FACTOR * y, (case, q, v, y)


def test_median_knob_in_every_build():
    """The median pass (MEDIAN_FILTERING 3 / 5 every MEDIAN_PERIOD iterations) is exact selection, so it is not a
    rounding departure: kernel 1 changes nothing, kernels 3 and 5 change the flow, in every build alike."""
    I0, I1 = _pair(97, 131, seed=8)
    P = gm.TVL1Params(nscales=2, warps=2, epsilon=0.0, iterations=10)
    base = nm.calc(I0, I1, P)
    assert _bits_equal(base, nm.calc(I0, I1, P, median=(1, 3)))
    m5 = nm.calc(I0, I1, P, median=(5, 3))
    assert not np.array_equal(base, m5)
    assert metrics.epe(m5, nm.calc(I0, I1, P, median=(5, 3), precision="f64")).max() <= 1e-3


@pytest.mark.parametrize("precision", ["f32", "eng"])
def test_result_independent_of_thread_count(eng_cr, precision):
    I0, I1 = _pair(97, 131, seed=9)
    P = gm.TVL1Params(nscales=3, warps=2, epsilon=0.01, iterations=30, gamma=0.5)
    n = nm.set_threads(0, precision)
    try:
        runs = []
        for t in sorted({1, 3, max(n, 2)}):
            nm.set_threads(t, precision)
            tr = []
            runs.append((nm.calc(I0, I1, P, trace=tr, precision=precision, median=(3, 4)), tr))
    finally:
        nm.set_threads(n, precision)
    for flow, tr in runs[1:]:
        assert _bits_equal(runs[0][0], flow) and tr == runs[0][1]
