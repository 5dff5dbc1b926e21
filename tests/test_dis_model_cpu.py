"""oracle/dis_model.py against the live cv2.DISOpticalFlow, stage by stage.

Bounds are measured (cv2 4.13, synthetic pairs of oracle.synth) and stated with their multiple:
* single level, propagation off (every patch independent), no refinement: with 1 and 4 descent steps the largest
  difference to cv2 is at most 4x the model's own float32-vs-float64 distance (measured 0.3x-0.4x); with the preset's 16
  steps the early stop can flip, so the 99th percentile is held to 4x the float64 distance's (measured 0.26x) and the
  share of pixels off by more than 1e-3 px to 0.2 % (measured 0.08 %);
* the refinement stage against cv2.VariationalRefinement with DIS's parameters: at most 4x the float64 distance
  (measured 1.4x);
* whole presets with propagation on (cv2's CPU propagation differs from the engine's OpenCL one): median endpoint
  difference at most 2x the measured 0.033 / 0.013 / 0.006 px, 99th percentile at most 2x the measured 0.15 / 0.056 /
  0.035 px, no pixel over 1 px (measured max 0.45), and the endpoint error to the known motion within 5 % + 0.005 px
  of cv2's (measured within 1.4 %).
"""
import cv2
import numpy as np
import pytest

from oracle import synth, dis_model as M, deepflow_model as DFM


def _cv2(I0, I1, p: M.DISParams):
    d = cv2.DISOpticalFlow_create(cv2.DISOPTICAL_FLOW_PRESET_FAST)
    d.setFinestScale(p.finest_scale)
    d.setCoarsestScale(p.coarsest_scale)
    d.setPatchSize(p.patch_size)
    d.setPatchStride(p.patch_stride)
    d.setGradientDescentIterations(p.grad_descent_iterations)
    d.setVariationalRefinementIterations(p.variational_refinement_iterations)
    d.setUseMeanNormalization(p.use_mean_normalization)
    d.setUseSpatialPropagation(p.use_spatial_propagation)
    return d.calc(I0, I1, None)


def test_presets_match_cv2():
    for pr in (0, 1, 2):
        d = cv2.DISOpticalFlow_create(pr)
        p = M.preset(pr)
        assert (d.getFinestScale(), d.getCoarsestScale(), d.getPatchSize(), d.getPatchStride(),
                d.getGradientDescentIterations(), d.getVariationalRefinementIterations()) == \
               (p.finest_scale, p.coarsest_scale, p.patch_size, p.patch_stride, p.grad_descent_iterations,
                p.variational_refinement_iterations)
        assert np.float32(d.getVariationalRefinementEpsilon()) == np.float32(p.epsilon)
        assert d.getDefaultName() == "my_object"


@pytest.mark.parametrize("shape", [(480, 640), (1080, 1920), (100, 100), (64, 200), (40, 40)])
def test_automatic_coarsest_scale(shape):
    """cv2's coarsest level is min(coarsestScale, the automatic rule): setting the rule's value (or more) changes
    nothing, one less does."""
    I0, I1, _ = synth.make_pair(*shape, seed=0)
    auto = M.auto_coarsest(*shape, 8)
    base = _cv2(I0, I1, M.DISParams(finest_scale=0))
    assert np.array_equal(base, _cv2(I0, I1, M.DISParams(finest_scale=0, coarsest_scale=auto)))
    assert np.array_equal(base, _cv2(I0, I1, M.DISParams(finest_scale=0, coarsest_scale=auto + 2)))
    if auto > 0:
        assert not np.array_equal(base, _cv2(I0, I1, M.DISParams(finest_scale=0, coarsest_scale=auto - 1)))


@pytest.mark.parametrize("shape,f", [((480, 640), 2), ((1080, 1920), 2), ((481, 643), 2), ((123, 457), 1),
                                     ((135, 240), 1), ((67, 120), 1), ((64, 64), 3)])
def test_pyramid_is_cv2_area_resize(shape, f):
    a = np.random.default_rng(1).integers(0, 256, shape, dtype=np.uint8)
    r, c = shape[0] >> f, shape[1] >> f
    assert np.array_equal(M.resize_area_u8(a, r, c), cv2.resize(a, (c, r), interpolation=cv2.INTER_AREA))
    r2, c2 = r // 2, c // 2
    b = cv2.resize(a, (c, r), interpolation=cv2.INTER_AREA)
    assert np.array_equal(M.resize_area_u8(b, r2, c2), cv2.resize(b, (c2, r2), interpolation=cv2.INTER_AREA))


def test_sobel_is_spatial_gradient():
    a = np.random.default_rng(0).integers(0, 256, (37, 53), dtype=np.uint8)
    gx, gy = cv2.spatialGradient(a)
    mx, my = M.sobel(a)
    assert np.array_equal(mx, gx) and np.array_equal(my, gy)


def test_refine_with_deepflow_epsilon_is_deepflow_model():
    I0, I1, gt = synth.make_pair(60, 80, seed=2, kind="smooth", mag=2.0)
    u, v = gt[..., 0] * np.float32(0.9), gt[..., 1] * np.float32(0.9)
    a = M.refine(I0.astype(np.float32), I1.astype(np.float32), u, v, 20, 5, 10, DFM.EPSILON, 1.6, 3, 5)
    b = DFM.refine(I0.astype(np.float32), I1.astype(np.float32), u, v, 20, 5, 10, 1.6, 3, 5)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("mean_norm", [True, False])
@pytest.mark.parametrize("gd", [1, 4, 16])
def test_single_level_search_vs_cv2(mean_norm, gd):
    I0, I1, _ = synth.make_pair(240, 320, seed=3, kind="smooth", mag=3.0)
    p = M.DISParams(finest_scale=0, coarsest_scale=0, grad_descent_iterations=gd, variational_refinement_iterations=0,
                    use_spatial_propagation=False, use_mean_normalization=mean_norm)
    ref = _cv2(I0, I1, p)
    a, b = M.calc(I0, I1, p), M.calc(I0, I1, p, dt=np.float64)
    d, r = np.abs(ref - a), np.abs(a - b)
    if gd < 16:
        assert d.max() <= 4 * r.max()
    else:
        assert np.quantile(d, 0.99) <= 4 * np.quantile(r, 0.99)
        assert (d > 1e-3).mean() <= 0.002


def test_refinement_stage_vs_cv2():
    I0, I1, _ = synth.make_pair(240, 320, seed=3, kind="smooth", mag=3.0)
    u0 = M.calc(I0, I1, M.DISParams(finest_scale=0, coarsest_scale=0, variational_refinement_iterations=0,
                                    use_spatial_propagation=False))
    vr = cv2.VariationalRefinement_create()
    vr.setAlpha(20)
    vr.setDelta(5)
    vr.setGamma(10)
    vr.setEpsilon(0.01)
    vr.setOmega(M.REFINE_OMEGA)
    vr.setSorIterations(M.REFINE_SOR_ITERATIONS)
    vr.setFixedPointIterations(5)
    ref = u0.copy()
    vr.calc(I0, I1, ref)
    args = (I0.astype(np.float32), I1.astype(np.float32), u0[..., 0], u0[..., 1], 20, 5, 10, 0.01, M.REFINE_OMEGA, 5,
            M.REFINE_SOR_ITERATIONS)
    a = np.stack(M.refine(*args), -1)
    b = np.stack(M.refine(*args, dt=np.float64), -1)
    assert np.abs(a - ref).max() <= 4 * np.abs(a - b).max()
    # and DIS's own refinement stage is that call: cv2's DIS with 5 refinement iterations is the call applied to its
    # output with none
    p0 = M.DISParams(finest_scale=0, coarsest_scale=0, use_spatial_propagation=False, variational_refinement_iterations=0)
    c0 = _cv2(I0, I1, p0)
    vr.calc(I0, I1, c0)
    assert np.array_equal(c0, _cv2(I0, I1, M.DISParams(finest_scale=0, coarsest_scale=0, use_spatial_propagation=False)))


@pytest.mark.parametrize("gd", [0, 16])
@pytest.mark.parametrize("prop", [False, True])
def test_initial_flow_single_level(gd, prop):
    """On one level cv2 starts each patch from the caller's flow at its centre, or from zero flow where zero's SSD is
    lower: with no descent and no propagation the model equals cv2 exactly; with them, as the searches above."""
    I0, I1, gt = synth.make_pair(240, 320, seed=3, kind="smooth", mag=3.0)
    F = (gt * np.float32(1.1)).astype(np.float32)
    p = M.DISParams(finest_scale=0, coarsest_scale=0, grad_descent_iterations=gd, variational_refinement_iterations=0,
                    use_spatial_propagation=prop)
    d = cv2.DISOpticalFlow_create(cv2.DISOPTICAL_FLOW_PRESET_FAST)
    d.setFinestScale(0)
    d.setCoarsestScale(0)
    d.setGradientDescentIterations(gd)
    d.setVariationalRefinementIterations(0)
    d.setUseSpatialPropagation(prop)
    ref = d.calc(I0, I1, F.copy())
    got = M.calc(I0, I1, p, flow=F)
    if gd == 0 and not prop:
        assert np.array_equal(got, ref)
    elif not prop:
        a, b = got, M.calc(I0, I1, p, dt=np.float64, flow=F)
        assert np.quantile(np.abs(got - ref), 0.99) <= 4 * np.quantile(np.abs(a - b), 0.99)
    else:  # cv2's CPU propagation: statistical, as the presets below
        assert np.median(np.linalg.norm(got - ref, axis=-1)) <= 0.07


MEASURED = M.CV2_MEASURED


@pytest.mark.parametrize("preset", [0, 1, 2])
@pytest.mark.parametrize("shape", [(480, 640), (1080, 1920)])
def test_presets_vs_cv2_statistical(preset, shape):
    I0, I1, gt = synth.make_pair(*shape, seed=1, kind="smooth", mag=4.0)
    ref = cv2.DISOpticalFlow_create(preset).calc(I0, I1, None)
    got = M.calc(I0, I1, M.preset(preset))
    e = np.linalg.norm(ref - got, axis=-1)
    q50, q99 = MEASURED[preset]
    assert np.median(e) <= 2 * q50 and np.quantile(e, 0.99) <= 2 * q99 and e.max() <= 1.0
    epe_ref, epe_got = np.linalg.norm(ref - gt, axis=-1).mean(), np.linalg.norm(got - gt, axis=-1).mean()
    assert epe_got <= 1.05 * epe_ref + 0.005


@pytest.mark.parametrize("kind", ["const", "affine", "smooth"])
def test_accuracy_on_known_motion(kind):
    I0, I1, gt = synth.make_pair(240, 320, seed=9, kind=kind, mag=3.0)
    for pr in (0, 1, 2):
        ref = cv2.DISOpticalFlow_create(pr).calc(I0, I1, None)
        got = M.calc(I0, I1, M.preset(pr))
        epe_ref, epe_got = np.linalg.norm(ref - gt, axis=-1).mean(), np.linalg.norm(got - gt, axis=-1).mean()
        assert epe_got <= 1.1 * epe_ref + 0.01, (pr, epe_got, epe_ref)
