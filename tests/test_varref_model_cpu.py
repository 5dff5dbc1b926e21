"""CPU checks of the VariationalRefinement model, oracle/dis_model.py ``refine`` (one calcUV call with epsilon as an
argument), against the live cv2.VariationalRefinement: per call, cv2's distance to the float64 model within a small
multiple of the float32 model's own distance to it, across parameters, input types, sizes and initial flows."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import dis_model as D  # noqa: E402

DEFAULTS = dict(fixed_point_iterations=5, sor_iterations=5, omega=1.6, alpha=20.0, delta=5.0, gamma=10.0,
                epsilon=0.001)
# the defaults and sets that move epsilon, omega and the iteration counts (tests/test_varref_gpu.py runs the same)
PARAM_SETS = [
    DEFAULTS,
    dict(DEFAULTS, epsilon=0.01),
    dict(DEFAULTS, omega=1.0, sor_iterations=12),
    dict(DEFAULTS, fixed_point_iterations=2, sor_iterations=25, omega=1.9, epsilon=0.05),
    dict(DEFAULTS, fixed_point_iterations=1, sor_iterations=1, alpha=3.0, delta=0.5, gamma=1.0),
]
SETTERS = dict(fixed_point_iterations="FixedPointIterations", sor_iterations="SorIterations", omega="Omega",
               alpha="Alpha", delta="Delta", gamma="Gamma", epsilon="Epsilon")


def pair(h, w, seed, u8=False):
    """A textured frame and a copy shifted by one column plus noise."""
    rng = np.random.default_rng(seed)
    I0 = rng.random((h, w)).astype(np.float32) * 255
    if h > 2 and w > 2:
        I0 = cv2.GaussianBlur(I0, (3, 3), 1.0)
    I1 = (np.roll(I0, 1, axis=1) + rng.random((h, w)).astype(np.float32) * 3).astype(np.float32)
    if u8:
        return np.rint(I0).astype(np.uint8), np.rint(np.clip(I1, 0, 255)).astype(np.uint8)
    return I0, I1


def initial_flow(h, w, kind, seed=7):
    """zero; small (a random field within +-1.5 px); big (the small field with a 6x6 block pointing 40, 200 and 1e4 px
    out of the image); out (every vector leaves the image)."""
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((h, w, 2), np.float32)
    f = ((rng.random((h, w, 2)) - 0.5) * 3).astype(np.float32)
    if kind == "big":
        for k, m in enumerate((40.0, 200.0, 1e4)):
            f[(k * 7) % h:(k * 7) % h + 6, (k * 11) % w:(k * 11) % w + 6] = (m, -m / 2)
    elif kind == "out":
        f = f + np.float32([w + 3.5, -(h + 2.25)])
    return f


def cv2_refine(I0, I1, flow, p):
    vr = cv2.VariationalRefinement_create()
    for k, v in p.items():
        getattr(vr, "set" + SETTERS[k])(v)
    return vr.calc(I0, I1, flow.copy())


def model(I0, I1, flow, p, dt):
    u, v = D.refine(I0, I1, flow[..., 0], flow[..., 1], p["alpha"], p["delta"], p["gamma"], p["epsilon"], p["omega"],
                    p["fixed_point_iterations"], p["sor_iterations"], dt)
    return np.stack([u, v], -1)


def check(I0, I1, flow, p):
    ref = cv2_refine(I0, I1, flow, p).astype(np.float64)
    m32 = model(I0, I1, flow, p, np.float32).astype(np.float64)
    m64 = model(I0, I1, flow, p, np.float64)
    own = np.abs(m32 - m64).max()
    err = np.abs(ref - m64).max()
    assert np.isfinite(ref).all() and np.isfinite(m32).all()
    assert err <= 4 * own + 1e-9, (err, own)


@pytest.mark.parametrize("p", PARAM_SETS, ids=range(len(PARAM_SETS)))
@pytest.mark.parametrize("kind", ["zero", "small", "big", "out"])
def test_model_matches_cv2_per_call(p, kind):
    I0, I1 = pair(40, 56, 3)
    check(I0, I1, initial_flow(40, 56, kind), p)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (7, 1), (2, 2), (3, 5), (1, 200), (200, 1), (2, 130), (65, 64),
                                 (120, 160), (240, 320)])
def test_model_matches_cv2_across_sizes(h, w):
    I0, I1 = pair(h, w, h * 1000 + w)
    check(I0, I1, initial_flow(h, w, "small"), DEFAULTS)


@pytest.mark.parametrize("kind", ["zero", "big"])
def test_u8_and_f32_inputs_alike(kind):
    """cv2 converts 8U frames to float without scaling: the u8 pair and its float copy give one result."""
    a, b = pair(33, 47, 9, u8=True)
    flow = initial_flow(33, 47, kind)
    got = cv2_refine(a, b, flow, DEFAULTS)
    assert np.array_equal(got, cv2_refine(a.astype(np.float32), b.astype(np.float32), flow, DEFAULTS))
    assert np.array_equal(model(a, b, flow, DEFAULTS, np.float32), model(a.astype(np.float32), b.astype(np.float32),
                                                                         flow, DEFAULTS, np.float32))
    check(a, b, flow, DEFAULTS)


@pytest.mark.parametrize("change", [dict(fixed_point_iterations=0), dict(fixed_point_iterations=-3),
                                    dict(sor_iterations=0), dict(sor_iterations=-1), dict(omega=0.0)])
def test_no_step_returns_the_flow_unchanged(change):
    I0, I1 = pair(30, 41, 4)
    flow = initial_flow(30, 41, "small")
    p = dict(DEFAULTS, **change)
    assert np.array_equal(cv2_refine(I0, I1, flow, p), flow)
    assert np.array_equal(model(I0, I1, flow, p, np.float32), flow)


def test_calc_uv_equals_calc():
    I0, I1 = pair(37, 52, 5)
    flow = initial_flow(37, 52, "small")
    vr = cv2.VariationalRefinement_create()
    u, v = vr.calcUV(I0, I1, flow[..., 0].copy(), flow[..., 1].copy())
    want = vr.calc(I0, I1, flow.copy())
    assert np.array_equal(u, want[..., 0]) and np.array_equal(v, want[..., 1])


def test_defaults_and_name():
    vr = cv2.VariationalRefinement_create()
    for k, v in DEFAULTS.items():
        assert getattr(vr, "get" + SETTERS[k])() == np.float32(v), k
    assert vr.getDefaultName() == "my_object"


def test_a_nan_in_the_flow_spreads_alike():
    """One NaN in the initial flow: cv2 and the model leave non-finite values at the same pixels (at this size, all)."""
    I0, I1 = pair(40, 56, 6)
    flow = initial_flow(40, 56, "small")
    flow[17, 23, 0] = np.nan
    ref = cv2_refine(I0, I1, flow, DEFAULTS)
    with np.errstate(invalid="ignore"):
        m32 = model(I0, I1, flow, DEFAULTS, np.float32)
    assert np.array_equal(np.isfinite(ref), np.isfinite(m32))
