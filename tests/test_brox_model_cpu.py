"""The Brox CUDA-semantics model: the C/OpenMP restatement (oracle/brox_model.c) equals the numpy statement
(oracle/brox_model.py) bit for bit, its correctly rounded rsqrt is correctly rounded for every float class, and the
perturbed mode is a fixed, bounded pattern.  The engine is compared with the C model in tests/test_brox_fullsize_gpu.py."""
import numpy as np
import pytest

from oracle import synth, brox_model as bm, brox_model_native as bn

pytestmark = pytest.mark.skipif(not bn.available(), reason="oracle/_build/libbrox_model.so not built")


def _pair(h, w, seed):
    if h >= 16 and w >= 16:
        I0, I1, _ = synth.make_pair(h, w, seed=seed, kind="smooth", dtype="f32")
        return I0, I1
    rng = np.random.default_rng(seed)
    return rng.random((h, w), dtype=np.float32), rng.random((h, w), dtype=np.float32)


@pytest.mark.parametrize("h,w,kw", [
    (1, 37, dict(inner_iterations=2, solver_iterations=3)),
    (37, 1, dict(inner_iterations=2, solver_iterations=3)),
    (2, 2, dict(inner_iterations=1, solver_iterations=1)),
    (16, 16, dict(inner_iterations=4, solver_iterations=2)),
    (45, 70, dict(scale_factor=0.5, inner_iterations=3, solver_iterations=4)),
    (41, 53, dict(scale_factor=0.95, outer_iterations=6, inner_iterations=2, solver_iterations=3)),
    (40, 56, dict(gamma=0.0, inner_iterations=2, solver_iterations=2)),
    (66, 97, dict(inner_iterations=1, solver_iterations=5)),
])
@pytest.mark.parametrize("rsqrt", bm.RSQRT_MODES)
def test_c_model_equals_numpy_model(h, w, kw, rsqrt):
    I0, I1 = _pair(h, w, seed=h * 131 + w)
    P = bm.BroxParams(**{**dict(outer_iterations=77), **kw})
    c_np, c_c = {}, {}
    a = bm.calc(I0, I1, P, rsqrt, c_np)
    b = bn.calc(I0, I1, P, rsqrt, c_c)
    assert np.isfinite(a).all()
    assert np.array_equal(a.view(np.int32), b.view(np.int32)), int((a != b).sum())
    assert c_np == c_c and c_c["levels"] == len(bm.pyramid_sizes(h, w, P.scale_factor, P.outer_iterations))
    assert c_c["mirrored"] > 0


def test_rsqrt_correctly_rounded_for_every_class():
    """1/sqrt(4x) = 1/sqrt(x) / 2 exactly, so the 2^24 mantissas at each exponent parity cover every normal float; the
    subnormals are all checked.  The criterion is exact integer arithmetic, independent of the helper's own check."""
    m = np.arange(1 << 23, dtype=np.uint32)
    for exp in (127, 128):
        x = ((np.uint32(exp) << np.uint32(23)) | m).view(np.float32)
        for i in range(0, x.size, 1 << 21):
            xs = x[i:i + (1 << 21)]
            assert bm.rsqrt_is_correctly_rounded(xs, bn.rsqrt_rn(xs)).all(), exp
    sub = np.arange(1, 1 << 23, dtype=np.uint32).view(np.float32)
    for i in range(0, sub.size, 1 << 21):
        xs = sub[i:i + (1 << 21)]
        assert bm.rsqrt_is_correctly_rounded(xs, bn.rsqrt_rn(xs)).all()
    # the numpy model's rsqrt and the double-rounding shortcut, on a sample
    xs = np.random.default_rng(0).random(1 << 16, dtype=np.float32) * np.float32(1e3) + np.float32(1e-6)
    assert np.array_equal(bm.rsqrt_rn(xs), bn.rsqrt_rn(xs))


def test_rsqrt_criterion_rejects_neighbours():
    x = np.array([2.0, 3.0, 1e-6, 1e-40, 7.5e30], np.float32)
    r = bn.rsqrt_rn(x)
    assert bm.rsqrt_is_correctly_rounded(x, r).all()
    assert not bm.rsqrt_is_correctly_rounded(x, np.nextafter(r, np.float32(0))).any()
    assert not bm.rsqrt_is_correctly_rounded(x, np.nextafter(r, np.float32(np.inf))).any()


def test_perturbed_mode_is_deterministic_and_within_two_ulp():
    k = bm.perturb_ulps(3, 2, 100000)
    assert np.array_equal(k, bm.perturb_ulps(3, 2, 100000))
    assert set(np.unique(k)) == {-2, -1, 0, 1, 2}
    assert not np.array_equal(k, bm.perturb_ulps(3, 1, 100000)) and not np.array_equal(k, bm.perturb_ulps(2, 2, 100000))
    r2 = np.random.default_rng(1).random(100000, dtype=np.float32) + np.float32(1e-6)
    e, p = bm.data_rsqrt(r2, "exact"), bm.data_rsqrt(r2, "perturbed", 3, 2)
    d = p.view(np.int32).astype(np.int64) - e.view(np.int32).astype(np.int64)
    assert np.array_equal(d, k)
    I0, I1 = _pair(40, 56, 4)
    P = bm.BroxParams(inner_iterations=2, outer_iterations=77, solver_iterations=2)
    a, b = bn.calc(I0, I1, P, "perturbed"), bn.calc(I0, I1, P, "perturbed")
    assert np.array_equal(a, b) and not np.array_equal(a, bn.calc(I0, I1, P, "exact"))


def test_model_recovers_synthetic_motion():
    I0, I1, gt = synth.make_pair(120, 160, seed=1, kind="const", dtype="f32")
    got = bn.calc(I0, I1, bm.BroxParams(inner_iterations=10, outer_iterations=77, solver_iterations=10))
    c = got[16:-16, 16:-16]
    assert abs(float(np.median(c[..., 0])) - 2.5) < 0.15 and abs(float(np.median(c[..., 1])) + 1.25) < 0.15
