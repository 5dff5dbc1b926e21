"""The interpolateFrames model's stages (oracle/interpolate_model.py): the engine's order against the reference's,
the order-free condition, the any-order error bound and its intervals, and the conversion and flush rules."""
import numpy as np

from oracle import synth, interpolate_model as im

F = np.float32


def _generic(h, w, seed):
    rng = np.random.default_rng(seed)
    f0, f1 = rng.random((h, w), dtype=F), rng.random((h, w), dtype=F)
    fl = synth.flow_field(h, w, "smooth", seed=seed) * F(1.7)
    bl = -fl + rng.normal(0, 0.3, (h, w, 2)).astype(F)
    return [f0, f1, fl[..., 0], fl[..., 1], bl[..., 0], bl[..., 1]]


def _dyadic(h, w, seed, step=0.125, lim=4.0):
    rng = np.random.default_rng(seed)
    f0, f1 = rng.random((h, w), dtype=F), rng.random((h, w), dtype=F)
    n = int(lim / step)
    return [f0, f1] + [(rng.integers(-n, n + 1, (h, w)) * step).astype(F) for _ in range(4)]


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def test_engine_order_equals_reference_order_in_corrected_mode():
    """Corrected mode accumulates every plane once in both orders: identical bits for any input."""
    for h, w, pitch in ((40, 56, 56), (33, 47, 64)):
        planes = _generic(h, w, h)
        for pos in (0.5, 0.2):
            a, A = im.interpolate_frames(*planes, pos, stride=pitch, corrected=True)
            b, B = im.interpolate_frames(*planes, pos, stride=pitch, corrected=True, order="engine")
            assert np.array_equal(_u32(a), _u32(b)) and np.array_equal(_u32(A), _u32(B))


def test_engine_order_equals_reference_order_where_the_reference_is_order_free():
    """Reference mode: with order-free accumulators, c + c equals the second accumulation of the coverage, and
    where c1 is a power of two the normalised bwdU is on the lattice too, so adding the bv splat to it at once
    or term by term gives the same bits.  Elsewhere the two orders are different computations."""
    h, w, pitch = 48, 60, 64  # rows 45.. lie past w*h: doubled coverage
    planes = _dyadic(h, w, 3, step=0.5, lim=2.0)
    con = im.splat(*planes[2:], 0.5, w, h, pitch)
    for p in im.PLANES:
        assert im.order_free(im.terms(con[p], h * pitch)).all(), p
    a, A = im.interpolate_frames(*planes, 0.5, stride=pitch, corrected=False)
    b, B = im.interpolate_frames(*planes, 0.5, stride=pitch, corrected=False, order="engine")
    A, B = A[:, :, :w], B[:, :, :w]
    for k in (0, 1, 2, 3, 5):
        assert np.array_equal(_u32(A[k]), _u32(B[k])), im.PLANES[k]
    c1 = im.accumulate(con["cov1"], h * pitch).reshape(h, pitch)[:, :w]
    m, _ = np.frexp(c1)
    pow2 = (np.abs(m) == 0.5) | (c1 == 0)
    assert pow2.mean() > 0.05 and (~pow2).mean() > 0.05
    assert np.array_equal(_u32(A[4][pow2]), _u32(B[4][pow2]))
    assert (A[4][~pow2] != B[4][~pow2]).any()
    # the output only differs through ur, in the second-frame-only branch
    second = im.blend_branches(A[0], A[1])[2]
    assert np.array_equal(_u32(a[~second]), _u32(b[~second]))


def test_lattice_and_order_free_condition_on_hand_built_contributions():
    idx = np.array([0, 0, 0, 2, 2, 3, 5], np.int64)
    val = np.array([0.5, 0.25, -0.125, 3 * 2.0 ** -10, 1.0, 0.0, 2.0 ** 20], F)
    t = im.terms(im.Contributions(idx, val), 6)
    assert t.count.tolist() == [3, 0, 2, 1, 0, 1]
    assert t.k.tolist() == [3, im.NO_LATTICE, 10, im.NO_LATTICE, im.NO_LATTICE, -20]
    assert t.abs_sum.tolist() == [0.875, 0, 1 + 3 * 2.0 ** -10, 0, 0, 2.0 ** 20]
    assert t.exact.tolist() == [0.625, 0, 1 + 3 * 2.0 ** -10, 0, 0, 2.0 ** 20]
    assert im.order_free(t).all()
    # on the 2^-24 lattice, magnitudes summing to 2^0 or more: not order-free
    t = im.terms(im.Contributions(np.zeros(3, np.int64), np.array([1.0, 2.0 ** -24, 2.0 ** -24], F)), 1)
    assert t.k.tolist() == [24] and not im.order_free(t)[0]
    # just below the limit: 2^23 + 2^22 + ... on the 2^0 lattice stays exact
    v = np.array([2.0 ** 23, 2.0 ** 22, 1.0, 1.0], F)
    assert im.order_free(im.terms(im.Contributions(np.zeros(4, np.int64), v), 1))[0]
    v = np.array([2.0 ** 23, 2.0 ** 23, 1.0], F)
    assert not im.order_free(im.terms(im.Contributions(np.zeros(3, np.int64), v), 1))[0]


def test_error_bound_covers_orders_that_change_the_float32_sum():
    val = np.array([1.0, 2.0 ** -24, 2.0 ** -24], F)
    exact = 1 + 2.0 ** -23
    sums = {}
    for order in ([0, 1, 2], [1, 2, 0]):
        c = im.Contributions(np.zeros(3, np.int64), val[order])
        sums[tuple(order)] = float(im.accumulate(c, 1)[0])
    assert sums[(0, 1, 2)] == 1.0 and sums[(1, 2, 0)] == exact  # the order changes the float32 sum
    t = im.terms(im.Contributions(np.zeros(3, np.int64), val), 1)
    assert t.exact[0] == exact
    B = im.error_bound(t)[0]
    assert all(abs(s - exact) <= B for s in sums.values())
    assert B < 2 * 2.0 ** -23  # and the bound is not loose: the worst order sits at half of it
    # a longer random sum: every permutation stays within the bound
    rng = np.random.default_rng(0)
    val = (rng.normal(0, 1, 200) * 10.0 ** rng.integers(-3, 3, 200)).astype(F)
    t = im.terms(im.Contributions(np.zeros(200, np.int64), val), 1)
    B = im.error_bound(t)[0]
    got = [float(im.accumulate(im.Contributions(np.zeros(200, np.int64), rng.permutation(val)), 1)[0])
           for _ in range(50)]
    assert len(set(got)) > 1 and max(abs(g - t.exact[0]) for g in got) <= B


def test_intervals_contain_any_order_of_the_atomics():
    """The engine-order model with its contributions shuffled stays inside normalised_intervals, both modes."""
    h, w, pitch = 40, 52, 64
    planes = _generic(h, w, 5)
    rng = np.random.default_rng(1)
    for corrected in (False, True):
        for pos in (0.5, 0.2):
            con = im.splat(*planes[2:], pos, w, h, pitch)
            T = {p: im.terms(con[p], h * pitch) for p in im.PLANES}
            iv = im.normalised_intervals(T, corrected, w, h, pitch)
            for trial in range(3):
                acc = []
                for p in im.PLANES:
                    o = rng.permutation(len(con[p].idx)) if trial else np.arange(len(con[p].idx))
                    acc.append(im.accumulate(im.Contributions(con[p].idx[o], con[p].val[o]), h * pitch))
                buf = im.normalise(acc, corrected, w, h, pitch).reshape(6, h, pitch)[:, :, :w]
                for k in range(6):
                    lo, hi = iv[k]
                    det = ~np.isnan(lo)
                    assert det.mean() > 0.99
                    assert ((buf[k] >= lo) & (buf[k] <= hi))[det].all(), (corrected, pos, k)
            # the intervals are tight: a one-ulp error in a normalised flow leaves them somewhere
            lo, hi = iv[4]
            assert (np.nextafter(buf[4], F(np.inf)) > hi).any()


def test_interval_of_a_coverage_that_may_be_zero_is_undetermined():
    # coverage 1 - 1 + 2^-30 (cancellation through the negative weights of the left-edge taps) -> undetermined;
    # no contributions at all -> c = 0 exactly, the engine divides by 1
    idx = np.array([0, 0, 0], np.int64)
    cov = im.Contributions(idx, np.array([1.0, -1.0, 2.0 ** -30], F))
    val = im.Contributions(idx, np.array([0.5, -0.5, 2.0 ** -31], F))
    none = im.Contributions(np.zeros(0, np.int64), np.zeros(0, F))
    T = {"cov0": im.terms(cov, 2), "cov1": im.terms(none, 2), "fwdU": im.terms(val, 2), "fwdV": im.terms(val, 2),
         "bwdU": im.terms(none, 2), "bwdV": im.terms(none, 2)}
    iv = im.normalised_intervals(T, True, 2, 1, 2)
    assert np.isnan(iv[2][0][0, 0]) and np.isnan(iv[3][1][0, 0])
    assert iv[2][0][0, 1] == iv[2][1][0, 1] == 0 and iv[4][0][0, 0] == iv[4][1][0, 0] == 0


def test_splat_coordinate_conversion_follows_ptx_cvt():
    """NaN -> 0: a NaN u sends its taps to column 0; an infinite u saturates and drops every tap."""
    h, w = 6, 8
    z = np.zeros((h, w), F)
    fu = z.copy()
    fu[3, 5] = np.nan
    fu[2, 4] = np.inf
    fu[4, 2] = -np.inf
    con = im.splat(fu, z, z, z, 0.5, w, h, w)
    taps_from = lambda c: c.idx[np.isnan(c.val)]
    # the NaN source at row 3: cy = 4 exactly, dy = 0 -> taps at rows 4 (weight NaN * 0) and 3 in column 0
    assert sorted(taps_from(con["fwdU"]).tolist()) == [3 * w, 4 * w]
    # zero flow elsewhere: every finite source puts weight 1 on its own pixel; the infinite sources put nothing
    # anywhere, and the NaN poisons the two column-0 pixels it reached
    cov = im.accumulate(con["cov0"], h * w).reshape(h, w)
    assert np.isnan(cov[3, 0]) and np.isnan(cov[4, 0]) and np.isfinite(cov).sum() == h * w - 2
    assert cov[2, 4] == cov[4, 2] == cov[3, 5] == 0
    assert cov[np.isfinite(cov)].sum() == h * w - 3 - 2


def test_atomics_flush_subnormal_contributions():
    """RED.ADD.F32.FTZ: a contribution value * weight below 2^-126 is added as 0."""
    h, w = 3, 4
    z = np.zeros((h, w), F)
    fu = np.full((h, w), 2.0 ** -125, F)  # normal; cx = j + 1 exactly, dx = 0
    fv = np.full((h, w), 0.5, F)          # dy = 0.25: the kept taps weigh 0.25 and 0.75
    con = im.splat(fu, fv, z, z, 0.5, w, h, w)
    raw = F(2.0 ** -125) * F(0.25)
    assert raw != 0 and abs(raw) < 2.0 ** -126  # subnormal before the atomic
    v = con["fwdU"].val
    assert not ((v != 0) & (np.abs(v) < 2.0 ** -126)).any()
    assert (v == F(2.0 ** -125) * F(0.75)).sum() == ((con["cov0"].val == 0.75)).sum() > 0
    assert (con["cov0"].val == 0.25).sum() > 0 and (v[con["cov0"].val == 0.25] == 0).all()
