"""CPU checks of oracle/sparselk_model.py, the CUDA-semantics model the SparsePyrLK engine is compared with bit for bit
(tests/test_sparselk_fullsize_gpu.py): its pyramid, both samplers and the block reduction against plain statements of
their definitions, the whole model against the live cv2.calcOpticalFlowPyrLK with the reference's own criterion, and
hand-built inputs for each early-return branch, each proven by its counter."""
import cv2
import numpy as np
import pytest

from oracle import synth, sparselk_model as sm

F = np.float32


@pytest.mark.parametrize("h,w", [(97, 131), (64, 80), (3, 2), (1, 7)])
def test_u8_pyramid_equals_cv2_pyrdown_except_at_ties(h, w):
    """Float rint rounds half to even where cv2's integer pyrDown rounds half up: the levels differ by exactly 1 at
    ties with an even floor and nowhere else.  The float sum of 8-bit inputs is exact, so the ties are exact."""
    rng = np.random.default_rng(h * w)
    img = rng.integers(0, 256, (h, w), dtype=np.uint8)
    img[: h // 2] = img[: h // 2] // 16 * 16  # coarse values make ties frequent
    exact = sm.pyr_down(img.astype(F))
    got = sm.pyramid(img, 1)[1][0]
    want = cv2.pyrDown(img).astype(F)
    assert got.shape == want.shape == ((h + 1) // 2, (w + 1) // 2)
    tie = exact - np.floor(exact) == 0.5
    even = np.floor(exact) % 2 == 0
    assert np.array_equal(got[~tie], want[~tie])
    assert np.array_equal(want[tie] - got[tie], even[tie].astype(F))
    if h > 8:
        assert (tie & even).sum() > 0


def _coords(n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    v = rng.uniform(lo, hi, n).astype(F)
    special = np.array([0, 0.5, -0.5, -1e-6, hi - 2 ** -8, -3.9, -4.1, -50, hi + 50, 1.5, 2.5], F)
    return np.concatenate([v, special])


@pytest.mark.parametrize("depth,norm", [(0, 255.0), (2, 65535.0), (5, 1.0)])
def test_texture_sampler_matches_its_definition(depth, norm):
    """8-bit weights floor(frac * 256 + 0.5) / 256 of the coordinate minus 0.5, clamped addresses, texels divided by
    the normalisation: evaluated here in float64, so only the float32 roundings of the blend differ."""
    rng = np.random.default_rng(depth)
    rows, cols = 9, 13
    hi = {0: 255, 2: 65535, 5: 1000}[depth]
    planes = rng.integers(0, hi + 1, (1, rows, cols)).astype(F)
    if depth == 5:
        planes = (planes * F(0.37)).astype(F)
    x = _coords(3000, -8, cols + 8, 1)
    y = np.random.default_rng(2).permutation(_coords(3000, -8, rows + 8, 3))
    got = sm.sample_tex(planes, y, x, norm)[0].astype(np.float64)

    def axis(c, n):
        b = c.astype(np.float64) - 0.5
        f = np.floor(b)
        a = np.floor((b - f) * 256 + 0.5) / 256
        i = np.clip(f, -2, n + 1).astype(int)
        return np.clip(i, 0, n - 1), np.clip(i + 1, 0, n - 1), a

    xa, xc, ax = axis(x, cols)
    ya, yc, ay = axis(y, rows)
    p = planes[0].astype(np.float64) / norm
    want = (1 - ax) * (1 - ay) * p[ya, xa] + ax * (1 - ay) * p[ya, xc] + (1 - ax) * ay * p[yc, xa] + ax * ay * p[yc, xc]
    assert np.all(np.abs(got - want) <= 4 * np.spacing(np.abs(want).astype(F)).astype(np.float64) + 1e-30)
    # the weights the model uses are multiples of 1/256 in [0, 1]
    _, _, a = sm.tex_axis(x, cols)
    assert np.array_equal(a * 256, np.round(a * 256)) and a.min() >= 0 and a.max() <= 1
    assert len(np.unique(a)) > 200


@pytest.mark.parametrize("depth", [0, 2, 4, 5])
def test_software_sampler_matches_its_definition(depth):
    """Exact weights from floor(x), zero outside the image, the coordinate clamped to [-4, n + 4], integer depths
    rounded half to even and saturated to the element type."""
    rng = np.random.default_rng(10 + depth)
    rows, cols = 7, 11
    lo, hi = {0: (0, 255), 2: (0, 65535), 4: (-2 ** 31, 2 ** 31 - 1), 5: (-1000, 1000)}[depth]
    planes = rng.integers(lo, hi, (2, rows, cols), endpoint=True).astype(F)
    x = _coords(3000, -8, cols + 8, 4)
    y = np.random.default_rng(5).permutation(_coords(3000, -8, rows + 8, 6))
    got = sm.sample_soft(planes, y, x, depth).astype(np.float64)
    xd, yd = x.astype(np.float64), y.astype(np.float64)
    x1 = np.floor(np.clip(xd, -4, cols + 4)).astype(int)
    y1 = np.floor(np.clip(yd, -4, rows + 4)).astype(int)
    for c in range(2):
        p = planes[c].astype(np.float64)

        def at(yy, xx):
            ok = (yy >= 0) & (yy < rows) & (xx >= 0) & (xx < cols)
            return np.where(ok, p[np.clip(yy, 0, rows - 1), np.clip(xx, 0, cols - 1)], 0.0)

        terms = [(x1 + 1 - xd) * (y1 + 1 - yd) * at(y1, x1), (xd - x1) * (y1 + 1 - yd) * at(y1, x1 + 1),
                 (x1 + 1 - xd) * (yd - y1) * at(y1 + 1, x1), (xd - x1) * (yd - y1) * at(y1 + 1, x1 + 1)]
        want = sum(terms)
        tol = sum(np.abs(t) for t in terms) * 1e-6 + 1e-9  # float32 roundings of the weights, products and sums
        if depth == 5:
            assert np.all(np.abs(got[c] - want) <= tol)
        else:
            lo_f, hi_f = sm.RANGES[depth]
            want = np.clip(want, lo_f, hi_f)
            near_half = np.abs(want - np.floor(want) - 0.5) <= tol
            r = np.rint(want)
            assert np.all((got[c] == r) | near_half)
            assert np.all(np.abs(got[c] - want) <= 0.5 + tol)
            assert np.array_equal(got[c], np.rint(got[c]))
        assert np.all(got[c][(xd < -1) | (xd > cols + 0) | (yd < -1) | (yd > rows + 0)] == 0)


def _reduce_loop(v):
    """block_sum written out: thread t adds elements t, t + 256, ... (channels inner), each warp's lane 0 folds
    16 / 8 / 4 / 2 / 1 lanes, the 8 warp sums are added in order."""
    E, C = v.shape
    acc = [F(0)] * 256
    for e in range(E):
        for c in range(C):
            acc[e % 256] = F(acc[e % 256] + v[e, c])
    warps = []
    for w in range(8):
        lanes = acc[32 * w:32 * w + 32]
        for o in (16, 8, 4, 2, 1):
            lanes = [F(lanes[i] + lanes[i + o]) for i in range(o)]
        warps.append(lanes[0])
    s = warps[0]
    for w in range(1, 8):
        s = F(s + warps[w])
    return s


@pytest.mark.parametrize("E,C", [(1, 1), (9, 3), (225, 1), (256, 4), (258, 1), (441, 3), (1000, 4)])
def test_block_sum_is_the_stated_order(E, C):
    rng = np.random.default_rng(E * 7 + C)
    v = (rng.standard_normal((5, E, C)) * np.exp(rng.uniform(-12, 12, (5, E, C)))).astype(F)
    got = sm.block_sum(v)
    for p in range(5):
        assert got[p].view(np.int32) == _reduce_loop(v[p]).view(np.int32)


def test_block_sum_order_differs_from_np_sum():
    """A constructed input on which the stated order and numpy's pairwise sum disagree: 2^24 is in thread 0's first
    element, and the 1.0s that follow it in thread 0 are each lost to rounding, while np.sum adds them first."""
    v = np.zeros((1, 1024, 1), F)
    v[0, 0, 0] = F(2 ** 24)
    v[0, 256::256, 0] = F(1)
    got = sm.block_sum(v)[0]
    assert got == _reduce_loop(v[0])
    assert got == F(2 ** 24) and np.sum(v) == F(2 ** 24 + 2)
    rng = np.random.default_rng(0)
    r = (rng.standard_normal((20, 441, 1)) * np.exp(rng.uniform(-10, 10, (20, 441, 1)))).astype(F)
    assert np.any(sm.block_sum(r) != np.sum(r, axis=(1, 2), dtype=F))


def _mismatch(a, sa, b, sb):
    bad = (sa.astype(bool) != sb.astype(bool))
    both = sa.astype(bool) & sb.astype(bool)
    bad |= both & (np.abs(a.astype(np.int32) - b.astype(np.int32)).max(axis=1) > 1)
    return bad.mean()


@pytest.mark.parametrize("cn", [1, 3])
def test_model_meets_the_reference_criterion(cn):
    """The whole model against the live CPU cv2.calcOpticalFlowPyrLK at the defaults (21x21, maxLevel 3, 30 iters),
    the reference's criterion: at most 1 % of the points differ in status or by more than one pixel
    (test_optflow.cpp:241-264).  Border features are masked as in tests/test_sparselk_gpu.py."""
    chans = [synth.make_pair(300, 400, seed=23 + 31 * c, kind="affine")[:2] for c in range(cn)]
    I0 = chans[0][0] if cn == 1 else np.stack([c[0] for c in chans], -1)
    I1 = chans[0][1] if cn == 1 else np.stack([c[1] for c in chans], -1)
    mask = np.zeros(I0.shape[:2], np.uint8)
    mask[12:-12, 12:-12] = 255
    gray = I0 if cn == 1 else np.ascontiguousarray(I0[..., 0])
    pts = cv2.goodFeaturesToTrack(gray, 600, 0.01, 0.0, mask=mask).reshape(-1, 2).astype(np.float32)
    assert len(pts) > 200
    gold, st_gold, err_gold = cv2.calcOpticalFlowPyrLK(I0, I1, pts.reshape(-1, 1, 2), None)
    nxt, status, err = sm.calc(I0, I1, pts)
    assert _mismatch(nxt, status, gold.reshape(-1, 2), st_gold.ravel()) <= 0.01
    ok = (status != 0) & (st_gold.ravel() != 0)
    assert np.isnan(err[status == 0]).all() and np.isfinite(err[status != 0]).all()
    # err on the texture path: the same mean absolute difference as cv2 on 8-bit values.  The software path (3
    # channels) rounds every sample to uchar first, so its err is a different quantity there.
    if cn == 1:
        assert abs(np.median(err[ok]) - np.median(err_gold.ravel()[ok])) < 0.05 * np.median(err_gold.ravel()[ok])


def _textured(h, w, seed=0):
    I0, I1, _ = synth.make_pair(h, w, seed=seed, kind="const")  # motion (2.5, -1.25)
    return I0, I1


def test_flat_image_gives_singular_points():
    flat = np.full((80, 100), 77, np.uint8)
    cnt = []
    nxt, status, err = sm.calc(flat, flat, np.array([[50.0, 40.0], [20.5, 30.25]], F), counters=cnt)
    assert all(c.singular == 2 for c in cnt) and (status == 0).all() and np.isnan(err).all()
    # never written: the initial estimate prevPts / 2^(maxLevel+1) stays
    assert np.array_equal(nxt, (np.array([[50.0, 40.0], [20.5, 30.25]], F) * F(1 / 16)).astype(F))


def test_points_outside_the_image_return_first():
    I0, I1 = _textured(80, 100)
    pts = np.array([[100.0, 40.0], [-1e-6, 40.0], [50.0, 80.0], [99.99, 79.99]], F)
    cnt = []
    nxt, status, _ = sm.calc(I0, I1, pts, counters=cnt)
    assert cnt[-1].outside_prev == 3 and status.tolist() == [0, 0, 0, 1]
    assert cnt[0].outside_prev == 2  # x = cols is inside level 3 (100 / 8 = 12.5 < 13 columns)
    # outside at level 0 means nothing was ever written for those points
    assert np.array_equal(nxt[1], (pts[1] * F(1 / 16)).astype(F))


def test_motion_that_leaves_the_image_drops_the_point():
    I0, I1 = _textured(80, 100)
    pts = np.array([[50.0, 0.3], [50.0, 0.6], [60.0, 1.0], [50.0, 40.0]], F)  # the motion carries the first ones up
    cnt = []
    _, status, _ = sm.calc(I0, I1, pts, counters=cnt)
    assert cnt[-1].left_during_iters > 0 and status[0] == 0 and status[-1] == 1


def test_iteration_counters():
    I0, I1 = _textured(80, 100)
    pts = np.array([[50.0, 40.0], [30.0, 30.0]], F)
    cnt = []
    sm.calc(I0, I1, pts, iters=0, counters=cnt)
    assert all(c.hit_iters == 2 and c.converged == 0 for c in cnt)
    cnt = []
    sm.calc(I0, I1, pts, counters=cnt)
    assert cnt[-1].converged == 2 and cnt[-1].hit_iters == 0


def test_use_initial_flow_starts_from_the_estimate():
    I0, I1 = _textured(120, 160)
    pts = np.array([[80.0, 60.0], [40.5, 70.25]], F)
    truth = (pts + F([2.5, -1.25])).astype(F)
    warm, status, _ = sm.calc(I0, I1, pts, max_level=0, next_pts=truth)
    assert (status == 1).all() and np.abs(warm - truth).max() < 0.1
    cold, _, _ = sm.calc(I0, I1, pts, max_level=0, iters=0)
    assert np.array_equal(cold, pts)  # zero iterations at one level: nextPts = prevPts / 2 * 2
