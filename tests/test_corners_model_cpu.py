"""CPU checks of oracle/corners_model.py against the live CPU reference (cv2.cornerHarris, cv2.cornerMinEigenVal,
cv2.goodFeaturesToTrack; the comparisons of modules/cudaimgproc/test/test_corners.cpp and test_gftt.cpp), and of its
literal sequential minDistance rule against a brute-force restatement."""
import cv2
import numpy as np
import pytest

from oracle import corners_model as M
from oracle import synth


def _img(rows, cols, seed, f32=False):
    a = np.clip(np.rint(synth.texture(rows, cols, seed)), 0, 255).astype(np.uint8)
    return (a / np.float32(255)).astype(np.float32) if f32 else a


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("border", [4, 1, 2])
def test_response_matches_cv2_over_the_reference_grid(f32, border):
    src = _img(240, 320, 11, f32)
    worst = 0.0
    for bs in (3, 5, 7):
        for ks in (0, 3, 5, 7):
            for harris in (False, True):
                got = M.response(src, bs, ks, border, harris)
                want = (cv2.cornerHarris(src, bs, ks, 0.04, borderType=border) if harris
                        else cv2.cornerMinEigenVal(src, bs, ksize=ks, borderType=border))
                worst = max(worst, float(np.abs(got - want).max()))
    assert worst <= 0.02, worst  # EXPECT_MAT_NEAR(..., 0.02)


def _mismatch(a, b):
    return float(np.mean(np.any(a.astype(np.int32) != b.astype(np.int32), axis=1)))


@pytest.mark.parametrize("md", [0.0, 3.0])
def test_gftt_matches_cv2_with_the_reference_criterion(md):
    img = _img(480, 640, 12)
    got, _ = M.gftt(img, 1000, 0.01, md)
    want = cv2.goodFeaturesToTrack(img, 1000, 0.01, md).reshape(-1, 2)
    assert len(got) == len(want) and _mismatch(got, want) <= 0.01


@pytest.mark.parametrize("kw", [dict(use_harris=True), dict(max_corners=0), dict(min_distance=2.4),
                                dict(min_distance=7.0, use_harris=True)])
def test_gftt_matches_cv2_harris_unlimited_fractional(kw):
    img = _img(240, 320, 13)
    p = dict(max_corners=500, quality_level=0.01, min_distance=0.0, block_size=3, use_harris=False, harris_k=0.04)
    p.update(kw)
    got, _ = M.gftt(img, **p)
    want = cv2.goodFeaturesToTrack(img, p["max_corners"], p["quality_level"], p["min_distance"],
                                   blockSize=3, useHarrisDetector=p["use_harris"], k=0.04).reshape(-1, 2)
    assert len(got) == len(want) and _mismatch(got, want) <= 0.01


def test_tie_order_equals_cv2():
    img = np.zeros((96, 128), np.uint8)
    for y in range(8, 88, 8):
        for x in range(8, 120, 8):
            img[y:y + 3, x:x + 3] = 200
    got, _ = M.gftt(img, 0, 0.01, 0.0)
    want = cv2.goodFeaturesToTrack(img, 0, 0.01, 0.0).reshape(-1, 2)
    assert len(got) > 50 and np.array_equal(got, want)


def _brute(pts, md, mc):
    cell = M.cv_round(md)
    out = []
    for p in pts.astype(np.float32):
        c = (int(p[0] / np.float32(cell)), int(p[1] / np.float32(cell)))
        ok = True
        for q in out:
            d = (int(q[0] / np.float32(cell)), int(q[1] / np.float32(cell)))
            dx, dy = p[0] - q[0], p[1] - q[1]
            if abs(c[0] - d[0]) <= 1 and abs(c[1] - d[1]) <= 1 and float(dx * dx + dy * dy) < md * md:
                ok = False
                break
        if ok:
            out.append(p)
            if mc > 0 and len(out) == mc:
                break
    return np.array(out, np.float32).reshape(-1, 2)


@pytest.mark.parametrize("seed", range(6))
def test_sequential_rule_equals_brute_force(seed):
    rng = np.random.default_rng(seed)
    pts = rng.integers(0, 60, (300, 2)).astype(np.float32)
    pts = np.unique(pts, axis=0)[rng.permutation(len(np.unique(pts, axis=0)))]
    for md in (1.0, 2.4, 3.0, 4.6, 10.0):
        for mc in (0, 1, 25):
            assert np.array_equal(M.select_sequential(pts, md, mc, 64, 64), _brute(pts, md, mc))


@pytest.mark.parametrize("md", [1.0, 1.5, 2.4, 2.5, 3.49, 10.0])
def test_two_cells_away_never_hides_a_conflict_on_integer_positions(md):
    # The grid looks only at the 3x3 cells around a corner.  Two cells apart means |dx| or |dy| >= cell + 1, and
    # cell = cvRound(minDistance) >= minDistance - 0.5, so on integer positions no conflict is ever two cells away:
    # the grid rule equals the plain distance rule, non-integer minDistance (2.4 -> cell 2) included.
    rng = np.random.default_rng(int(md * 10))
    pts = np.unique(rng.integers(0, 40, (400, 2)), axis=0).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]
    out = []
    for p in pts:
        if all(float((p[0] - q[0]) ** 2 + (p[1] - q[1]) ** 2) >= md * md for q in out):
            out.append(p)
    assert np.array_equal(M.select_sequential(pts, md, 0, 40, 40), np.array(out, np.float32).reshape(-1, 2))
