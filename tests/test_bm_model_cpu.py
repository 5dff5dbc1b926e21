"""CPU checks of oracle/bm_model.py, the statement of cudalegacy's block-matching flows that the bm.cu engine is held to
bit for bit: FastOpticalFlowBM's closed-form SAD against a literal restatement of the reference's per-tile sliding sums,
its tie order, the cudev border rule, the spiral scan table and the grid function's per-cell branches."""
import numpy as np
import pytest

from oracle import bm_model as M

INT_MAX = 2**31 - 1


# ------------------------------------------------------------------------------------------------ FastBM
def tile_algorithm(I0, I1, sw, bw):
    """The reference kernel's own order of work (src/cuda/bm_fast.cu): 128x32 tiles, a block_window-entry column ring per
    candidate, column sums carried down from the tile row above, each of 128 threads scanning t, t+128, ... for its
    first strict minimum, and reduceKeyVal<128>'s merges: within each warp over lanes 16, 8, 4, 2, 1, then over the four
    warp results 2, 1, the lower position keeping ties."""
    sr, br = sw // 2, bw // 2
    b = sr + br
    E0, E1 = M.pad_cudev(I0, b).astype(np.int64), M.pad_cudev(I1, b).astype(np.int64)
    rows, cols = I0.shape
    n = sw * sw
    idx = np.arange(n)
    cy, cx = idx // sw - sr, idx % sw - sr

    def a(y, x):
        return E0[y + b, x + b]

    def bv(y, x):  # I1 at per-candidate coordinates
        return E1[y + b, x + b]

    out = np.zeros((rows, cols, 2), np.float32)
    for tby in range(0, rows, 32):
        up = {}
        for tbx in range(0, cols, 128):
            ring = np.zeros((bw, n), np.int64)
            dist = np.zeros(n, np.int64)
            first = 0
            for i in range(tby, min(tby + 32, rows)):
                for j in range(tbx, min(tbx + 128, cols)):
                    if j == tbx:
                        dist[:] = 0
                        for tx in range(-br, br + 1):
                            col = np.zeros(n, np.int64)
                            for ty in range(-br, br + 1):
                                col += np.abs(a(i + ty, j + tx) - bv(i + cy + ty, j + cx + tx))
                            dist += col
                            ring[tx + br] = col
                        up[j] = ring[bw - 1].copy()
                        first = 0
                    else:
                        if i == tby:
                            col = np.zeros(n, np.int64)
                            for ty in range(-br, br + 1):
                                col += np.abs(a(i + ty, j + br) - bv(i + cy + ty, j + cx + br))
                        else:
                            col = (up[j] + np.abs(a(i + br, j + br) - bv(i + cy + br, j + cx + br))
                                   - np.abs(a(i - br - 1, j + br) - bv(i + cy - br - 1, j + cx + br)))
                        dist += col - ring[first]
                        ring[first] = col
                        up[j] = col
                        first = (first + 1) % bw
                    # per-thread strided scan, then the merge tree
                    key = np.full(128, INT_MAX, np.int64)
                    ind = np.full(128, -1, np.int64)
                    for t in range(min(128, n)):
                        seg = dist[t::128]
                        q = int(np.argmin(seg))  # argmin returns the first minimum
                        key[t], ind[t] = seg[q], t + 128 * q
                    key, ind = key.reshape(4, 32), ind.reshape(4, 32)
                    for s in (16, 8, 4, 2, 1):
                        take = key[:, s:2 * s] < key[:, :s]
                        key[:, :s] = np.where(take, key[:, s:2 * s], key[:, :s])
                        ind[:, :s] = np.where(take, ind[:, s:2 * s], ind[:, :s])
                    wk, wi = key[:, 0].copy(), ind[:, 0].copy()
                    for s in (2, 1):
                        take = wk[s:2 * s] < wk[:s]
                        wk[:s] = np.where(take, wk[s:2 * s], wk[:s])
                        wi[:s] = np.where(take, wi[s:2 * s], wi[:s])
                    out[i, j] = (wi[0] % sw - sr, wi[0] // sw - sr)
    return out


@pytest.mark.parametrize("bw", [1, 3, 7])
@pytest.mark.parametrize("sw", [1, 2, 21])
def test_closed_form_equals_the_reference_sliding_sums(sw, bw):
    rng = np.random.default_rng(sw * 10 + bw)
    rows, cols = 34, 259  # two tile rows, three tile columns
    I0 = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
    I1 = np.roll(I0, (1, -2), (0, 1))
    I1 = np.where(rng.random(I1.shape) < 0.2, rng.integers(0, 256, I1.shape), I1).astype(np.uint8)
    if sw == 21:  # quantised frames: many exact ties between candidates
        I0, I1 = (I0 // 128 * 128).astype(np.uint8), (I1 // 128 * 128).astype(np.uint8)
    assert np.array_equal(M.fastbm(I0, I1, sw, bw), tile_algorithm(I0, I1, sw, bw))


TIE_SHIFT = (0, 3)


def tie_frames(sw, period, shift):
    rng = np.random.default_rng(3)
    tile = rng.integers(0, 256, (period, period), dtype=np.uint8)
    I0 = np.tile(tile, (64 // period + 2, 96 // period + 2))[:64, :96]
    I1 = np.roll(I0, shift, (0, 1))
    return I0, I1


def tie_winner(sw, period, shift):
    """Offsets of the winners by the reference's order, by lowest k and by (k mod 128, k div 128) among the zero-SAD
    candidates of a periodic pair."""
    sr = sw // 2
    ks = [k for k in range(sw * sw) if (k // sw - sr - shift[0]) % period == 0 and (k % sw - sr - shift[1]) % period == 0]
    ref = min(ks, key=lambda k: (int(M.tie_pref(k % 128)), k // 128))
    plain = min(ks, key=lambda k: (k % 128, k // 128))
    off = lambda k: (k % sw - sr, k // sw - sr)
    return off(ref), off(min(ks)), off(plain), len(ks)


def test_tie_pref_is_the_merge_tree_order():
    assert sorted(M.tie_pref(np.arange(128)).tolist()) == list(range(128))
    assert np.array_equal(M.tie_pref(M.tie_pref(np.arange(128))), np.arange(128))  # its own inverse
    assert M.tie_pref(0) == 0 and M.tie_pref(32) == 64 and M.tie_pref(64) == 32 and M.tie_pref(1) == 16
    assert M.tie_pref(2) < M.tie_pref(1)  # thread 2 meets thread 0's slot before thread 1 does


def test_tie_order_follows_the_reference_reduction():
    sw, period, shift = 21, 7, TIE_SHIFT
    ref, low, plain, n = tie_winner(sw, period, shift)
    assert n > 1 and ref != low and ref != plain  # the designed pair separates the orders
    I0, I1 = tie_frames(sw, period, shift)
    f = M.fastbm(I0, I1, sw, 3)
    inner = f[16:-16, 16:-16]  # away from the reflected border the pattern is exactly periodic
    assert (inner[..., 0] == ref[0]).all() and (inner[..., 1] == ref[1]).all()
    assert not ((inner[..., 0] == low[0]) & (inner[..., 1] == low[1])).any()
    assert M.rank(130, 21) < M.rank(5, 21)  # a tie between k = 5 and k = 130 goes to 130


@pytest.mark.parametrize("sw", [1, 2, 21])
def test_flat_frames_give_minus_sr(sw):
    I = np.full((9, 40), 77, np.uint8)
    f = M.fastbm(I, I, sw, 7)
    assert (f == -(sw // 2)).all()


def brd_base_reflect101(i, n):
    """cudev BrdBase<BrdReflect101>: idx_low(idx_high(i)), written out with the scalar operators."""
    last = n - 1
    hi = abs(last - abs(last - i)) % n
    return abs(hi) % n


@pytest.mark.parametrize("shape", [(1, 1), (1, 37), (37, 1), (5, 5)])
def test_border_follows_the_cudev_fold(shape):
    import cv2
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    b = 21 // 2 + 7 // 2
    got = M.pad_cudev(img, b)
    want = np.array([[img[brd_base_reflect101(y, shape[0]), brd_base_reflect101(x, shape[1])]
                      for x in range(-b, shape[1] + b)] for y in range(-b, shape[0] + b)])
    assert np.array_equal(got, want)
    if shape == (5, 5):  # the CPU's iterative rule differs once the border exceeds the frame
        assert not np.array_equal(got, cv2.copyMakeBorder(img, b, b, b, b, cv2.BORDER_REFLECT_101))


def test_key_layout_sides():
    assert M.key_layout(21, 7) == (9, False)
    assert not M.key_layout(109, 21)[1] and M.key_layout(109, 23)[1]
    assert not M.key_layout(21, 31)[1]
    assert not M.check_fastbm_args(21, 8) and not M.check_fastbm_args(110, 7) and not M.check_fastbm_args(21, 33)
    assert M.check_fastbm_args(109, 31) and M.check_fastbm_args(2, 1)


# ------------------------------------------------------------------------------------------------ grid BM
@pytest.mark.parametrize("W,H", [(3, 3), (2, 5), (5, 2), (0, 0), (0, 3), (4, 0)])
def test_spiral_table(W, H):
    t = M.spiral(W, H)
    assert len(t) == (2 * W + 1) * (2 * H + 1) - 1
    assert len({tuple(p) for p in t}) == len(t)
    assert {tuple(p) for p in t} == {(x, y) for x in range(-W, W + 1) for y in range(-H, H + 1)} - {(0, 0)}
    m = min(W, H)
    ring = np.maximum(np.abs(t[:, 0]), np.abs(t[:, 1]))[:4 * m * (m + 1)]
    assert (np.diff(ring) >= 0).all()
    for r in range(1, m + 1):
        seg = t[4 * (r - 1) * r:4 * r * (r + 1)]
        assert tuple(seg[0]) == (-r + 1, -r) and tuple(seg[-1]) == (-r, -r)
        assert (np.abs(np.diff(seg, axis=0)).sum(1) == 1).all()  # a connected clockwise walk
    rest = t[4 * m * (m + 1):]
    if W < H:
        assert (np.abs(rest[:, 1]) > m).all()
    elif W > H:
        assert (np.abs(rest[:, 0]) > m).all()


def test_frames_are_swapped():
    rng = np.random.default_rng(0)
    prev = rng.integers(0, 256, (64, 80), dtype=np.uint8)
    curr = np.roll(prev, (2, 3), (0, 1))  # curr is prev shifted by +s
    vx, vy = M.calc_bm(prev, curr, (8, 8), (8, 8), (4, 4), False)
    inner = (slice(1, -1), slice(1, -1))
    assert (vx[inner] == -3).all() and (vy[inner] == -2).all()


def test_float2int_rn():
    v = np.array([0.5, 1.5, 2.5, -0.5, -1.5, 0.49999997, 1e10, -1e10, np.nan, np.inf, -np.inf], np.float32)
    assert M.float2int_rn(v).tolist() == [0, 2, 2, 0, -2, 0, INT_MAX, -2**31, 0, INT_MAX, -2**31]


def test_int32_wrap():
    assert M.wrap32(8 + INT_MAX) == -2**31 + 7
    assert M.wrap32(-2**31 - 1) == INT_MAX
    prev = np.random.default_rng(0).integers(0, 256, (32, 32), dtype=np.uint8)
    vx = np.full((3, 3), 3e9, np.float32)  # saturates to INT_MAX; every X1 + offset wraps out of range
    c = {}
    gx, gy = M.calc_bm(prev, prev, (16, 16), (8, 8), (2, 2), True, vx, np.zeros_like(vx), counters=c)
    assert (gx == np.float32(INT_MAX)).all() and (gy == 0).all() and c["escaped"] == 9


def branch_case(name):
    rng = np.random.default_rng(5)
    tex = rng.integers(0, 256, (48, 64), dtype=np.uint8)
    if name == "accepted_at_start":
        return tex, tex, False, None
    if name == "accepted_in_search":
        return tex, np.roll(tex, (1, -2), (0, 1)), False, None
    if name == "best_of_scan":
        return tex, rng.integers(0, 256, tex.shape, dtype=np.uint8), False, None
    if name == "tie_averaged":
        return np.full(tex.shape, 100, np.uint8), np.full(tex.shape, 110, np.uint8), False, None
    if name == "escaped":
        return np.zeros(tex.shape, np.uint8), np.full(tex.shape, 255, np.uint8), False, None
    # the start lies one column left of the frame; the first in-range candidate matches exactly and is accepted, but
    # everything before it (nothing) was worse than escapeLevel, so the start is kept
    vr, vc = M.vel_size(48, 64, (16, 16), (8, 8))
    vx = -(np.arange(vc, dtype=np.float32) * 8 + 1)[None, :].repeat(vr, 0)
    return tex, tex, True, (vx, np.zeros_like(vx))


@pytest.mark.parametrize("name", M.BRANCHES)
def test_every_branch_is_reached(name):
    prev, curr, use_prev, vel = branch_case(name)
    c = {}
    args = (vel[0], vel[1]) if vel else (None, None)
    vx, vy = M.calc_bm(prev, curr, (16, 16), (8, 8), (3, 3), use_prev, *args, counters=c)
    assert c[name] > 0, c
    if name == "escaped_after_accept":
        assert vx[0, 0] == -1 and vy[0, 0] == 0  # cell (0, 0): nothing in range precedes the exact match
    if name == "tie_averaged":
        assert (c["tie_averaged"] == vx.size)


def test_vel_size_uses_c_division():
    assert M.vel_size(48, 64, (16, 16), (8, 8)) == (5, 7)
    assert M.vel_size(10, 10, (16, 16), (8, 8)) == (0, 0)  # -6 / 8 truncates to 0
    assert M.vel_size(10, 10, (11, 11), (8, 8)) == (0, 0)
