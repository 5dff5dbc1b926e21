"""oracle/lkpyramid_model.py against the live cv2.calcOpticalFlowPyrLK / cv2.buildOpticalFlowPyramid, bit for bit:
uint32 views of nextPts and err (where cv2 writes err), status exact.  Also the new C-ABI symbols' presence."""
import os

import cv2
import numpy as np
import pytest

from oracle import lkpyramid_model as M
from oracle import synth

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(rows, cols, cn=1, seed=1, shift=(2, 1), flat=False):
    a = np.clip(np.rint(synth.texture(rows, cols, seed)), 0, 255).astype(np.uint8)
    if flat:
        a[rows // 3: 2 * rows // 3, cols // 3: 2 * cols // 3] = 128
    if cn > 1:
        a = np.stack([a, np.roll(a, 3, 1), np.roll(a, 5, 0), a[::-1]][:cn], -1).copy()
    b = cv2.GaussianBlur(np.roll(a, shift, (0, 1)), (3, 3), 0.8)
    return a, b.reshape(a.shape)


def grid(rows, cols, step=4.3, margin=-3.0):
    xs = np.arange(margin, cols - margin, step)
    ys = np.arange(margin, rows - margin, step * 0.87)
    return np.stack(np.meshgrid(xs, ys), -1).reshape(-1, 1, 2).astype(np.float32)


def compare(I0, I1, pts, init=None, prev=None, nxt=None, **kw):
    cvkw = dict(winSize=kw.get("win_size", (21, 21)), maxLevel=kw.get("max_level", 3),
                criteria=kw.get("criteria", (3, 30, 0.01)), flags=kw.get("flags", 0),
                minEigThreshold=kw.get("min_eig_threshold", 1e-4))
    g, s, e = cv2.calcOpticalFlowPyrLK(I0, I1, pts, None if init is None else init.copy(), **cvkw)
    cnt = {}
    o, st, er, wr = M.calc(I0 if prev is None else prev, I1 if nxt is None else nxt, pts, init, counters=cnt, **kw)
    assert np.array_equal(st, s.ravel())
    assert np.array_equal(o.view(np.uint32), g.reshape(-1, 2).view(np.uint32))
    assert np.array_equal(er[wr].view(np.uint32), e.ravel()[wr].view(np.uint32))
    return cnt


@pytest.mark.parametrize("shape", [(1, 1), (1, 40), (40, 1), (2, 3), (7, 300), (300, 9), (61, 83), (240, 320), (480, 640)])
def test_sizes(shape):
    I0, I1 = frames(*shape, seed=3)
    pts = grid(*shape, step=max(shape) / 40 + 0.7)
    compare(I0, I1, pts, win_size=(5, 5), max_level=3)


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("win", [(3, 3), (21, 21), (31, 31), (9, 17)])
def test_channels_and_windows(cn, win):
    I0, I1 = frames(97, 131, cn)
    compare(I0, I1, grid(97, 131, 5.1), win_size=win, max_level=2)


@pytest.mark.parametrize("max_level", [0, 3, 9])
def test_levels(max_level):
    I0, I1 = frames(120, 160, shift=(5, -4))
    compare(I0, I1, grid(120, 160, 6.3), max_level=max_level, win_size=(15, 15))


@pytest.mark.parametrize("ctype", [1, 2, 3])
@pytest.mark.parametrize("iters", [0, 1, 100])
def test_criteria(ctype, iters):
    I0, I1 = frames(96, 128, shift=(3, 2))
    compare(I0, I1, grid(96, 128, 5.7), criteria=(ctype, iters, 0.03), win_size=(11, 11))


@pytest.mark.parametrize("thr", [0.0, 1e-4, 1e-1])
def test_min_eig_threshold_and_flat_regions(thr):
    I0, I1 = frames(120, 160, flat=True)
    cnt = compare(I0, I1, grid(120, 160, 3.9), min_eig_threshold=thr, win_size=(9, 9))
    if thr > 0:
        assert cnt["rejected_mineig"] > 0


def test_flags():
    I0, I1 = frames(120, 160, 3, shift=(4, 3))
    pts = grid(120, 160, 6.1)
    init = (pts + np.float32(2.5)).astype(np.float32)
    compare(I0, I1, pts, init=init, flags=M.OPTFLOW_USE_INITIAL_FLOW, win_size=(13, 13))
    compare(I0, I1, pts, flags=M.OPTFLOW_LK_GET_MIN_EIGENVALS, win_size=(13, 13))


def test_gftt_points_border_and_outside():
    I0, I1 = frames(240, 320, shift=(6, -5))
    gf = cv2.goodFeaturesToTrack(I0, 500, 0.01, 5).astype(np.float32)
    edge = np.array([[[0, 0]], [[319.5, 239.5]], [[-10.5, 5]], [[5, 260]], [[-40, -40]], [[1e9, 3]], [[319.99, 0.01]]],
                    np.float32)
    compare(I0, I1, np.concatenate([gf, edge]), win_size=(21, 21))


def test_1080p():
    I0, I1 = frames(1080, 1920, shift=(3, 4))
    gf = cv2.goodFeaturesToTrack(I0, 2000, 0.01, 5).astype(np.float32)
    compare(I0, I1, gf)


def test_pyramid_inputs_equal_image_inputs():
    I0, I1 = frames(120, 160, shift=(3, 2))
    pts = grid(120, 160, 5.3)
    _, P0 = M.build_pyramid(I0, (25, 25), 3, True)
    _, P1 = M.build_pyramid(I1, (21, 21), 3, False)
    _, Q0 = M.build_pyramid(I0, (21, 21), 1, False)
    compare(I0, I1, pts, prev=P0, nxt=P1)
    compare(I0, I1, pts, prev=Q0, nxt=I1, max_level=1)  # cv2 with maxLevel 1 = pyramid's cap
    compare(I0, I1, pts, prev=I0, nxt=P1)


@pytest.mark.parametrize("shape,cn,win,ml", [((480, 640), 1, (21, 21), 3), ((61, 83), 3, (5, 7), 4), ((5, 9), 4, (3, 3), 3),
                                             ((1, 1), 1, (3, 3), 2)])
@pytest.mark.parametrize("deriv", [True, False])
def test_build_pyramid_matches_cv2(shape, cn, win, ml, deriv):
    I0, _ = frames(*shape, cn=cn)
    n, want = cv2.buildOpticalFlowPyramid(I0, win, ml, withDerivatives=deriv)
    m, P = M.build_pyramid(I0, win, ml, deriv)
    assert n == m
    step = 2 if deriv else 1
    assert len(want) == (m + 1) * step
    bw, bh = win
    for lv in range(m + 1):
        img = want[lv * step].reshape(P.interior(lv).shape)
        assert np.array_equal(P.interior(lv), img)
        # the border: what cv2.copyMakeBorder makes of cv2's level
        bordered = cv2.copyMakeBorder(img, bh, bh, bw, bw, cv2.BORDER_REFLECT_101).reshape(P.levels[lv].shape)
        assert np.array_equal(P.levels[lv], bordered)
        if deriv:
            d = want[lv * step + 1].reshape(P.interior(lv, True).shape)
            assert np.array_equal(P.interior(lv, True), d)
            assert not P.derivs[lv][:bh].any() and not P.derivs[lv][:, :bw].any()


def test_every_branch_fired():
    """Flat texture, a 3x3 window, points on and outside the border: each per-point rule fires and still matches cv2."""
    I0, I1 = frames(120, 160, flat=True, shift=(5, -4))
    edge = np.array([[[-10.5, 5]], [[5, 130]], [[-40, -40]], [[1e9, 3]], [[159.9, 119.9]]], np.float32)
    pts = np.concatenate([grid(120, 160, 3.3), edge])
    cnt = compare(I0, I1, pts, win_size=(3, 3), max_level=3)
    for k, v in compare(I0, I1, pts, win_size=(9, 9), max_level=2, min_eig_threshold=1e-2).items():
        cnt[k] += v
    for k in ("out_of_image", "rejected_mineig", "out_of_window", "eps_stop", "half_step"):
        assert cnt[k] > 0, (k, cnt)


def test_abi_declares_and_binds_the_tracker():
    from opencv_contrib_b200 import _lib
    names = {n for n, _, _ in _lib.SYMBOLS}
    want = {"b2f_lkpyr_default_params", "b2f_lkpyr_create", "b2f_lkpyr_set_params", "b2f_lkpyr_get_params",
            "b2f_lkpyr_build_pyramid", "b2f_lkpyr_pyramid_level", "b2f_lkpyr_pyramid_info", "b2f_lkpyr_calc",
            "b2f_lkpyr_destroy", "b2f_lkpyr_last_cuda_error", "b2f_lkpyr_engine", "b2f_lkpyr_pyramid_create",
            "b2f_lkpyr_pyramid_destroy"}
    assert want <= names
    hdr = open(os.path.join(_ROOT, "include", "b200flow.h")).read()
    for n in want:
        assert n + "(" in hdr, n
    if os.path.exists(_lib.LIB_PATH):
        _lib.lib()  # binds every symbol or raises
