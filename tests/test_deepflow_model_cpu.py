"""CPU checks of the DeepFlow oracles: oracle/deepflow_model.py against the live cv2.VariationalRefinement per call, the
pyramid of oracle/deepflow_ref.py against the reference's level counts, and the full pipeline against cv2's own
last-bit sensitivity."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import synth, metrics, deepflow_ref as R, deepflow_model as M  # noqa: E402


def _pair(h, w, seed):
    rng = np.random.default_rng(seed)
    I0 = cv2.GaussianBlur(rng.random((h, w)).astype(np.float32) * 255, (3, 3), 1.0)
    I1 = (np.roll(I0, 1, axis=1) + rng.random((h, w)).astype(np.float32) * 3).astype(np.float32)
    return I0, I1


@pytest.mark.parametrize("h,w", [(13, 17), (31, 26), (40, 9)])
@pytest.mark.parametrize("fp,sor", [(1, 0), (1, 1), (1, 25), (5, 1), (5, 25)])
@pytest.mark.parametrize("init", [0.0, 1.5])
def test_model_matches_cv2_variational_refinement(h, w, fp, sor, init):
    """One VariationalRefinement call: model vs cv2 within a small multiple of the model's own float32-vs-float64
    distance."""
    I0, I1 = _pair(h, w, h * 100 + w)
    flow = ((np.random.default_rng(7).random((h, w, 2)) - 0.5) * 2 * init).astype(np.float32)
    sp = dict(R.solver_params(R.DeepFlowParams()), fixed_point_iterations=fp, sor_iterations=sor)
    ref = R.cv2_solver(I0, I1, flow, sp).astype(np.float64)
    m32 = M.model_solver(np.float32)(I0, I1, flow, sp).astype(np.float64)
    m64 = M.model_solver(np.float64)(I0, I1, flow, sp)
    own = np.abs(m32 - m64).max()
    err = np.abs(ref - m64).max()
    assert err <= 4 * own + 1e-9, (err, own)
    if sor == 0:
        assert np.array_equal(m32, flow.astype(np.float64))


def test_model_uses_u8_and_f32_inputs_alike():
    I0, I1 = _pair(21, 23, 5)
    a, b = np.rint(I0).astype(np.uint8), np.rint(np.clip(I1, 0, 255)).astype(np.uint8)
    sp = dict(R.solver_params(R.DeepFlowParams()), fixed_point_iterations=2, sor_iterations=3)
    flow = np.zeros((21, 23, 2), np.float32)
    ref = R.cv2_solver(a, b, flow, sp)
    got = M.model_solver()(a, b, flow, sp)
    assert np.abs(ref - got).max() < 1e-5


@pytest.mark.parametrize("rows,cols,levels", [(1080, 1920, 74), (480, 640, 59), (26, 100, 1), (27, 27, 2)])
def test_pyramid_level_counts(rows, cols, levels):
    sizes = R.pyramid_sizes(rows, cols)
    assert len(sizes) == levels
    assert all(min(s) > 25 for s in sizes[1:])


@pytest.mark.parametrize("max_layers,levels", [(0, 1), (1, 2), (5, 6)])
def test_max_layers_counts_levels_below_the_source(max_layers, levels):
    """buildPyramid pushes the source, then adds at most maxLayers levels."""
    assert len(R.pyramid_sizes(480, 640, R.DeepFlowParams(max_layers=max_layers))) == levels


def test_blur_and_resize_follow_cv2():
    rng = np.random.default_rng(3)
    I = (rng.random((37, 29)) * 255).astype(np.float32)
    k0, k1 = M.gaussian_taps(0.6)
    # the reference's sigma is the float member 0.6f, widened to double
    kern = cv2.getGaussianKernel(3, float(np.float32(0.6)), ktype=cv2.CV_32F).ravel()
    assert (k1, k0, k1) == tuple(float(x) for x in kern)
    sg = float(np.float32(0.6))
    assert np.abs(M.blur3(I, k0, k1) - cv2.GaussianBlur(I, (3, 3), sg, sigmaY=sg)).max() <= 1e-6 * 255 * 4
    for r, c in ((35, 28), (39, 31), (18, 14)):
        want = cv2.resize(I, (c, r), interpolation=cv2.INTER_LINEAR)
        assert np.abs(M.resize_linear(I, r, c) - want).max() <= 1e-6 * 255 * 4


def test_driver_with_model_solver_matches_restatement():
    """The restated driver over cv2's VariationalRefinement vs the same driver over the model's solver, and the
    model's own pipeline (its blur and resize) vs cv2: both within cv2's own distance under a 1e-6 perturbation of I1
    (the solver differs from cv2's only by float rounding per call, which the pyramid amplifies like the perturbation)."""
    I0, I1, _ = synth.make_pair(48, 64, seed=3, kind="const")
    a, mean_y, p99_y = _yardstick(I0, I1)
    for got in (R.calc(I0, I1, solver=M.model_solver()), M.calc(I0, I1)):
        e = metrics.epe(got, a)
        assert e.mean() <= mean_y and np.quantile(e, 0.99) <= p99_y, (e.mean(), mean_y, np.quantile(e, 0.99), p99_y)


def _yardstick(I0, I1):
    """cv2 DeepFlow vs cv2 DeepFlow of I1 perturbed by 1e-6 relative: the pipeline's own last-bit sensitivity."""
    base = R.calc(I0, I1)
    pert = (I1.astype(np.float32) * np.float32(1 + 1e-6)).astype(np.float32)
    e = metrics.epe(R.calc(I0, pert), base)
    return base, float(e.mean()), float(np.quantile(e, 0.99))


def test_model_pipeline_within_cv2_sensitivity():
    I0, I1, _ = synth.make_pair(96, 120, seed=5, kind="smooth", mag=3.0)
    base, mean_y, p99_y = _yardstick(I0, I1)
    e = metrics.epe(M.calc(I0, I1), base)
    assert e.mean() <= 4 * mean_y and np.quantile(e, 0.99) <= 4 * p99_y, (e.mean(), mean_y, np.quantile(e, 0.99), p99_y)
