"""oracle/optflowgf_model.py against the live cv2 on its portable path (setUseOptimized(False), IPP off), bit for bit:
uint32 views of every primitive's output and of whole calcOpticalFlowFarneback calls; and the model against default
cv2 within 4x cv2's own default-vs-portable distance."""
import cv2
import numpy as np
import pytest

from oracle import optflowgf_model as M
from oracle import synth


@pytest.fixture
def portable():
    opt, ipp = cv2.useOptimized(), cv2.ipp.useIPP()
    cv2.setUseOptimized(False)
    cv2.ipp.setUseIPP(False)
    yield
    cv2.setUseOptimized(opt)
    cv2.ipp.setUseIPP(ipp)


def neq(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape
    return int((a.view(np.uint32) != b.view(np.uint32)).sum())


def pair(rows, cols, seed=0, shift=(1, 2)):
    a = synth.texture(rows, cols, seed)
    b = np.roll(a, shift, (0, 1))
    return np.clip(np.rint(a), 0, 255).astype(np.uint8), np.clip(np.rint(b), 0, 255).astype(np.uint8)


def run(a, b, flow, *args):
    c = cv2.calcOpticalFlowFarneback(a, b, None if flow is None else flow.copy(), *args)
    m = M.calc(a, b, flow, *args)
    assert neq(c, m) == 0
    return c


# ------------------------------------------------------------------------------------------------------ primitives


@pytest.mark.parametrize("ks,sigma", [(3, 0), (5, 0), (7, 0), (3, 0.5), (5, 1.2), (9, 1.5), (13, 2.5), (39, 7.5), (83, 16.4)])
def test_gaussian_kernel_and_blur(portable, ks, sigma):
    assert neq(cv2.getGaussianKernel(ks, sigma, ktype=cv2.CV_32F).ravel(), M.gaussian_kernel(ks, sigma)) == 0
    rng = np.random.default_rng(ks)
    for shape in [(97, 131), (ks, ks + 2), (240, 320)]:
        a = (rng.standard_normal(shape) * 80).astype(np.float32)
        assert neq(cv2.GaussianBlur(a, (ks, ks), sigma, sigmaY=sigma), M.gaussian_blur(a, ks, sigma)) == 0


RESIZES = [((123, 157), (61, 79)), ((123, 157), (31, 39)), ((30, 40), (60, 80)), ((61, 79), (123, 157)),
           ((60, 80), (30, 40)), ((62, 86), (31, 43)), ((10, 90), (5, 45)), ((68, 120), (135, 240)), ((480, 640), (60, 80))]


@pytest.mark.parametrize("cn", [1, 2])
@pytest.mark.parametrize("src,dst", RESIZES)
def test_resize_linear(portable, cn, src, dst):
    a = (np.random.default_rng(1).standard_normal(src + ((cn,) if cn > 1 else ())) * 30).astype(np.float32)
    assert neq(cv2.resize(a, dst[::-1], interpolation=cv2.INTER_LINEAR), M.resize_linear(a, *dst)) == 0


@pytest.mark.parametrize("cn", [1, 2])
@pytest.mark.parametrize("src,dst", [((123, 157), (61, 79)), ((480, 640), (60, 80)), ((62, 86), (31, 43)),
                                     ((480, 640), (30, 40)), ((1080, 1920), (34, 60)), ((99, 64), (33, 16)),
                                     ((97, 131), (97, 131)), ((200, 300), (41, 33))])
def test_resize_area(portable, cn, src, dst):
    a = (np.random.default_rng(2).standard_normal(src + ((cn,) if cn > 1 else ())) * 30).astype(np.float32)
    assert neq(cv2.resize(a, dst[::-1], interpolation=cv2.INTER_AREA), M.resize_area(a, *dst)) == 0


@pytest.mark.parametrize("n,sigma", [(5, 1.1), (7, 1.5), (3, 1.1), (6, 1.3), (5, 0.0), (9, 2.0)])
def test_cholesky_tables(n, sigma):
    """the 6x6 Cholesky inverse restated here equals cv::invert(DECOMP_CHOLESKY) on FarnebackPrepareGaussian's G"""
    if sigma < float(np.finfo(np.float32).eps):
        sigma = n * 0.3
    g = [np.float32(np.exp(-x * x / (2 * sigma * sigma))) for x in range(-n, n + 1)]
    s = 1.0 / sum(float(v) for v in g)
    g = [np.float32(float(v) * s) for v in g]
    G = np.zeros((6, 6))
    f32 = np.float32
    for y in range(-n, n + 1):
        for x in range(-n, n + 1):
            gyx = f32(g[y + n] * g[x + n])
            G[0, 0] += float(gyx)
            G[1, 1] += float(f32(f32(gyx * f32(x)) * f32(x)))
            G[3, 3] += float(f32(f32(f32(f32(gyx * f32(x)) * f32(x)) * f32(x)) * f32(x)))
            G[5, 5] += float(f32(f32(f32(f32(gyx * f32(x)) * f32(x)) * f32(y)) * f32(y)))
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    _, inv = cv2.invert(G, flags=cv2.DECOMP_CHOLESKY)
    ours = np.array(M._chol_inv(G.tolist()))
    assert np.array_equal(inv.view(np.uint64), ours.view(np.uint64))


# ------------------------------------------------------------------------------------------------------ whole calls

BASE = (0.5, 5, 13, 10, 5, 1.1, 0)


@pytest.mark.parametrize("shape", [(1, 1), (1, 37), (37, 1), (3, 4), (9, 12), (31, 31), (32, 32), (33, 33), (63, 64),
                                   (64, 65), (65, 63), (12, 200), (97, 131), (480, 640)])
def test_sizes(portable, shape):
    a, b = pair(*shape)
    run(a, b, None, *BASE)
    run(a, b, None, 0.5, 5, 13, 3, 5, 1.1, M.OPTFLOW_FARNEBACK_GAUSSIAN)


@pytest.mark.parametrize("args", [
    (0.8, 5, 13, 3, 5, 1.1, 0), (0.3, 5, 13, 3, 5, 1.1, 0), (0.0, 5, 13, 3, 5, 1.1, 0), (-0.5, 3, 13, 2, 5, 1.1, 0),
    (0.5, 0, 13, 3, 5, 1.1, 0), (0.5, 1, 13, 3, 5, 1.1, 0), (0.5, 3, 13, 3, 5, 1.1, 0), (0.5, -2, 13, 3, 5, 1.1, 0),
    (0.5, 5, 1, 3, 5, 1.1, 0), (0.5, 5, 2, 3, 5, 1.1, 0), (0.5, 5, 14, 3, 5, 1.1, 0), (0.5, 5, 31, 3, 5, 1.1, 0),
    (0.5, 5, 13, 0, 5, 1.1, 0), (0.5, 5, 13, 1, 5, 1.1, 0), (0.5, 5, 13, 2, 5, 1.1, 0), (0.5, 5, 13, 10, 5, 1.1, 0),
    (0.5, 5, 13, 3, 7, 1.5, 0), (0.5, 5, 13, 3, 3, 1.1, 0), (0.5, 5, 13, 3, 6, 1.3, 0), (0.5, 5, 13, 3, 5, 0.0, 0),
    (0.5, 5, 1, 3, 5, 1.1, 256), (0.5, 5, 2, 3, 5, 1.1, 256), (0.5, 5, 14, 3, 7, 1.5, 256), (0.5, 5, 31, 2, 5, 1.1, 256),
    (0.8, 5, 5, 10, 6, 0.0, 256)])
def test_parameters(portable, args):
    a, b = pair(97, 131, seed=3, shift=(2, -3))
    run(a, b, None, *args)


@pytest.mark.parametrize("rows", [30, 63, 64, 65, 129])
@pytest.mark.parametrize("iters", [2, 3])
def test_interleaved_update_heights(portable, rows, iters):
    """cv2 updates M in stripes of max(1024 / width, winSize) rows during the next solve; a full pass is the same"""
    a, b = pair(rows, 40, seed=rows)
    run(a, b, None, 0.5, 0, 5, iters, 5, 1.1, 0)
    run(a, b, None, 0.5, 0, 5, iters, 5, 1.1, 256)


def initial_flows(rows, cols):
    ys, xs = np.mgrid[0:rows, 0:cols].astype(np.float32)
    smooth = synth.flow_field(rows, cols, "smooth", seed=1, mag=4.0)
    return {"zero": np.zeros((rows, cols, 2), np.float32), "smooth": smooth,
            "huge": np.full((rows, cols, 2), 1e4, np.float32),
            "out": np.stack([-xs - 5, (rows - ys) + 3], -1).astype(np.float32),
            "neg_zero": np.full((rows, cols, 2), -0.0, np.float32)}


@pytest.mark.parametrize("kind", ["zero", "smooth", "huge", "out", "neg_zero"])
@pytest.mark.parametrize("flags", [4, 4 | 256])
@pytest.mark.parametrize("shape,levels", [((97, 131), 5), ((128, 160), 5), ((97, 131), 0), ((120, 150), 2)])
def test_initial_flow(portable, kind, flags, shape, levels):
    a, b = pair(*shape, seed=5)
    run(a, b, initial_flows(*shape)[kind], 0.5, levels, 9, 2, 5, 1.1, flags)


def test_initial_flow_pyr_scale_08(portable):
    a, b = pair(100, 140, seed=6)
    run(a, b, initial_flows(100, 140)["smooth"], 0.8, 5, 9, 2, 5, 1.1, 4)


def test_depths_and_float_range(portable):
    a, b = pair(97, 131, seed=7)
    c8 = run(a, b, None, *BASE)
    for t in (np.uint16, np.float32):
        assert neq(c8, cv2.calcOpticalFlowFarneback(a.astype(t), b.astype(t), None, *BASE)) == 0
    rng = np.random.default_rng(8)
    fa = (a.astype(np.float32) * 3.7 - 300) + rng.standard_normal(a.shape).astype(np.float32)
    fb = (b.astype(np.float32) * 3.7 - 300)
    run(fa, fb, None, *BASE)


def test_fast_pyramids_ignored_and_class_equals_function(portable):
    a, b = pair(97, 131, seed=9)
    c = cv2.calcOpticalFlowFarneback(a, b, None, *BASE)
    for fast in (False, True):
        o = cv2.FarnebackOpticalFlow_create(5, 0.5, fast, 13, 10, 5, 1.1, 0)
        assert o.getDefaultName() == "DenseOpticalFlow.FarnebackOpticalFlow"
        assert neq(c, o.calc(a, b, None)) == 0


def test_threads_do_not_change_the_result(portable):
    a, b = pair(240, 320, seed=10)
    n = cv2.getNumThreads()
    try:
        cv2.setNumThreads(1)
        one = cv2.calcOpticalFlowFarneback(a, b, None, *BASE)
    finally:
        cv2.setNumThreads(n)
    assert neq(one, cv2.calcOpticalFlowFarneback(a, b, None, *BASE)) == 0


def default_distance(a, b, args, flow=None):
    """endpoint distance between default cv2 and the model, and cv2's own default-vs-portable distance"""
    opt, ipp = cv2.useOptimized(), cv2.ipp.useIPP()
    cv2.setUseOptimized(True)
    cv2.ipp.setUseIPP(True)
    try:
        d = cv2.calcOpticalFlowFarneback(a, b, None if flow is None else flow.copy(), *args)
    finally:
        cv2.setUseOptimized(opt)
        cv2.ipp.setUseIPP(ipp)
    cv2.setUseOptimized(False)
    cv2.ipp.setUseIPP(False)
    try:
        p = cv2.calcOpticalFlowFarneback(a, b, None if flow is None else flow.copy(), *args)
    finally:
        cv2.setUseOptimized(opt)
        cv2.ipp.setUseIPP(ipp)
    m = M.calc(a, b, flow, *args)
    return np.linalg.norm(d - m, axis=-1), np.linalg.norm(d - p, axis=-1)


@pytest.mark.parametrize("flags", [0, 256])
def test_model_close_to_default_cv2(flags):
    a, b = pair(480, 640, seed=0, shift=(3, -2))
    ours, theirs = default_distance(a, b, (0.5, 5, 13, 10, 5, 1.1, flags))
    assert ours.mean() <= 4 * theirs.mean() + 1e-12
    assert np.quantile(ours, 0.99) <= 4 * np.quantile(theirs, 0.99) + 1e-12
    assert ours.max() <= 4 * theirs.max() + 1e-12
