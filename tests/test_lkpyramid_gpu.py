"""The video module's calcOpticalFlowPyrLK / buildOpticalFlowPyramid on the GPU (csrc/lkpyramid.cu) against
oracle/lkpyramid_model.py and the live cv2, bit for bit: uint32 views of nextPts and err, status exact."""
import cv2
import numpy as np
import pytest
import torch

import opencv_contrib_b200 as ocb
from opencv_contrib_b200 import lkpyramid as LK
from oracle import lkpyramid_model as M
from oracle import synth

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


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


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def check(got, I0, I1, pts, init=None, prev=None, nxt=None, against_cv2=True, **kw):
    o, s, e = (x.cpu().numpy() for x in got)
    want, st, er, wr = M.calc(I0 if prev is None else prev, I1 if nxt is None else nxt, pts, init, **kw)
    assert np.array_equal(s.ravel(), st)
    assert np.array_equal(o.reshape(-1, 2).view(np.uint32), want.view(np.uint32))
    assert np.array_equal(e.ravel()[wr].view(np.uint32), er[wr].view(np.uint32))
    if against_cv2:
        g, cs, ce = cv2.calcOpticalFlowPyrLK(I0, I1, pts, None if init is None else init.copy(),
                                             winSize=kw.get("win_size", (21, 21)), maxLevel=kw.get("max_level", 3),
                                             criteria=kw.get("criteria", (3, 30, 0.01)), flags=kw.get("flags", 0),
                                             minEigThreshold=kw.get("min_eig_threshold", 1e-4))
        assert np.array_equal(o.reshape(-1, 2).view(np.uint32), g.reshape(-1, 2).view(np.uint32))
        assert np.array_equal(s.ravel(), cs.ravel())


def run(I0, I1, pts, init=None, **kw):
    args = dict(winSize=kw.get("win_size", (21, 21)), maxLevel=kw.get("max_level", 3),
                criteria=kw.get("criteria", (3, 30, 0.01)), flags=kw.get("flags", 0),
                minEigThreshold=kw.get("min_eig_threshold", 1e-4))
    return ocb.calcOpticalFlowPyrLK(t(I0), t(I1), t(pts), None if init is None else t(init), **args)


@pytest.mark.parametrize("shape", [(1, 1), (1, 40), (40, 1), (2, 3), (7, 300), (300, 9), (61, 83), (240, 320), (480, 640)])
def test_sizes(shape):
    I0, I1 = frames(*shape, seed=3)
    pts = grid(*shape, step=max(shape) / 40 + 0.7)
    check(run(I0, I1, pts, win_size=(5, 5)), I0, I1, pts, win_size=(5, 5))


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("win", [(3, 3), (21, 21), (31, 31), (9, 17)])
def test_channels_and_windows(cn, win):
    I0, I1 = frames(97, 131, cn)
    pts = grid(97, 131, 5.1)
    check(run(I0, I1, pts, win_size=win, max_level=2), I0, I1, pts, win_size=win, max_level=2)


@pytest.mark.parametrize("max_level", [0, 3, 9])
@pytest.mark.parametrize("ctype,iters", [(1, 0), (1, 1), (2, 100), (3, 100), (3, 30)])
def test_levels_and_criteria(max_level, ctype, iters):
    I0, I1 = frames(120, 160, shift=(5, -4))
    pts = grid(120, 160, 6.3)
    kw = dict(max_level=max_level, win_size=(15, 15), criteria=(ctype, iters, 0.03))
    check(run(I0, I1, pts, **kw), I0, I1, pts, **kw)


@pytest.mark.parametrize("thr", [0.0, 1e-4, 1e-1])
@pytest.mark.parametrize("flags", [0, M.OPTFLOW_LK_GET_MIN_EIGENVALS, M.OPTFLOW_USE_INITIAL_FLOW])
def test_thresholds_flags_flat(thr, flags):
    I0, I1 = frames(120, 160, 3, flat=True, shift=(4, 3))
    pts = grid(120, 160, 3.9)
    init = (pts + np.float32(2.5)).astype(np.float32) if flags & M.OPTFLOW_USE_INITIAL_FLOW else None
    kw = dict(min_eig_threshold=thr, win_size=(9, 9), flags=flags)
    check(run(I0, I1, pts, init, **kw), I0, I1, pts, init, **kw)


def test_1080p_gftt_and_grid():
    I0, I1 = frames(1080, 1920, shift=(3, 4))
    gf = cv2.goodFeaturesToTrack(I0, 2000, 0.01, 5).astype(np.float32)
    check(run(I0, I1, gf), I0, I1, gf)
    g = grid(1080, 1920, 15.2, 2.0)[:10000]
    assert len(g) == 10000
    check(run(I0, I1, g), I0, I1, g, against_cv2=False)


@pytest.mark.parametrize("n", [1, 31, 33, 70000])
def test_point_counts(n):
    I0, I1 = frames(240, 320, shift=(2, -3))
    rng = np.random.default_rng(n)
    pts = (rng.random((n, 1, 2)) * np.array([330, 250]) - 5).astype(np.float32)
    check(run(I0, I1, pts, win_size=(7, 7)), I0, I1, pts, win_size=(7, 7), against_cv2=n < 1000)


def test_large_window_has_no_limit():
    # the tracker keeps no patch in shared memory, so any window cv2 accepts runs
    I0, I1 = frames(200, 260)
    pts = grid(200, 260, 17.0)
    check(run(I0, I1, pts, win_size=(81, 65), max_level=1), I0, I1, pts, win_size=(81, 65), max_level=1)


def test_pitched_roi_frames():
    big0, big1 = frames(150, 210, 3)
    a, b = t(big0)[10:130, 7:187], t(big1)[10:130, 7:187]
    I0, I1 = big0[10:130, 7:187].copy(), big1[10:130, 7:187].copy()
    pts = grid(120, 180, 5.5)
    got = ocb.calcOpticalFlowPyrLK(a, b, t(pts), None, winSize=(11, 11))
    check(got, I0, I1, pts, win_size=(11, 11))


def test_gftt_detect_output_feeds_in():
    I0, I1 = frames(480, 640, shift=(3, -2))
    det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, 3.0)
    corners = det.detect(t(I0))
    got = ocb.calcOpticalFlowPyrLK(t(I0), t(I1), corners, None)
    pts = corners.cpu().numpy()
    check(got, I0, I1, pts)
    assert got[0].shape == corners.shape


def test_handle_reused_across_sizes_and_two_streams():
    lk = LK.SparsePyrLKOpticalFlow_create((11, 11), 3)
    for shape in [(240, 320), (61, 83), (480, 640), (61, 83)]:
        I0, I1 = frames(*shape, seed=5)
        pts = grid(*shape, 6.7)
        check(lk.calc(t(I0), t(I1), t(pts)), I0, I1, pts, win_size=(11, 11))
    lk2 = LK.SparsePyrLKOpticalFlow_create((11, 11), 3)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    A0, A1 = frames(240, 320, seed=6)
    B0, B1 = frames(300, 200, 3, seed=7)
    pa, pb = grid(240, 320, 4.1), grid(300, 200, 4.3)
    ta = [t(x) for x in (A0, A1, pa)]
    tb = [t(x) for x in (B0, B1, pb)]
    torch.cuda.synchronize()
    for _ in range(3):
        with torch.cuda.stream(s1):
            ra = lk.calc(*ta, stream=s1)
        with torch.cuda.stream(s2):
            rb = lk2.calc(*tb, stream=s2)
    torch.cuda.synchronize()
    check(ra, A0, A1, pa, win_size=(11, 11))
    check(rb, B0, B1, pb, win_size=(11, 11))
    assert lk.getActivePath() & 0xff == 1


def test_pyramid_reused_across_three_pairs():
    seq = [frames(240, 320, seed=8, shift=(k, -k))[1] for k in range(4)]
    pts = grid(240, 320, 5.9)
    lk = LK.SparsePyrLKOpticalFlow_create((15, 15), 3)
    _, prev = LK.buildOpticalFlowPyramid(t(seq[0]), (15, 15), 3)
    for k in range(1, 4):
        _, nxt = LK.buildOpticalFlowPyramid(t(seq[k]), (15, 15), 3)
        got = [x.clone() for x in lk.calc(prev, nxt, t(pts))]
        fresh = lk.calc(t(seq[k - 1]), t(seq[k]), t(pts))
        for a, b in zip(got, fresh):
            assert np.array_equal(a.cpu().numpy().view(np.uint8), b.cpu().numpy().view(np.uint8))
        check(got, seq[k - 1], seq[k], pts, win_size=(15, 15))
        prev = nxt


@pytest.mark.parametrize("deriv", [True, False])
@pytest.mark.parametrize("shape,cn,win,ml", [((480, 640), 1, (21, 21), 3), ((61, 83), 3, (5, 7), 4), ((1, 1), 1, (3, 3), 2)])
def test_build_pyramid_matches_cv2(shape, cn, win, ml, deriv):
    I0, _ = frames(*shape, cn=cn)
    n, want = cv2.buildOpticalFlowPyramid(I0, win, ml, withDerivatives=deriv)
    m, P = LK.buildOpticalFlowPyramid(t(I0), win, ml, withDerivatives=deriv)
    assert n == m and len(P) == m + 1
    lst = P.tolist()
    assert len(lst) == len(want)
    bw, bh = win
    for k, (g, w) in enumerate(zip(lst, want)):
        g = g.cpu().numpy()
        assert np.array_equal(g.reshape(w.shape), w)
        pad = P.padded(k // (2 if deriv else 1), deriv and k % 2 == 1).cpu().numpy()
        if deriv and k % 2:
            assert not pad[:bh].any() and not pad[-bh:].any() and not pad[:, :bw].any() and not pad[:, -bw:].any()
        else:
            assert np.array_equal(pad.reshape(-1), cv2.copyMakeBorder(w, bh, bh, bw, bw, cv2.BORDER_REFLECT_101).reshape(-1))


def test_pyramid_without_derivatives_as_prev_and_level_caps():
    I0, I1 = frames(240, 320, shift=(4, 4))
    pts = grid(240, 320, 6.1)
    _, P0 = LK.buildOpticalFlowPyramid(t(I0), (25, 25), 1, withDerivatives=False)
    got = ocb.calcOpticalFlowPyrLK(P0, t(I1), t(pts), None, maxLevel=3)
    check(got, I0, I1, pts, max_level=1)  # the pyramid's level count caps maxLevel


def test_refusals():
    I0, I1 = frames(60, 80)
    with pytest.raises(ocb.B2FError) as e:
        LK.buildOpticalFlowPyramid(t(I0), (9, 9), 2, pyrBorder=cv2.BORDER_REPLICATE)
    assert e.value.status == 2
    with pytest.raises(ocb.B2FError) as e:
        LK.buildOpticalFlowPyramid(t(I0), (9, 9), 2, derivBorder=cv2.BORDER_REFLECT_101)
    assert e.value.status == 2
    _, small = LK.buildOpticalFlowPyramid(t(I0), (5, 5), 2)
    with pytest.raises(ocb.B2FError) as e:  # a border narrower than the window
        ocb.calcOpticalFlowPyrLK(small, t(I1), t(grid(60, 80)), None, winSize=(9, 9))
    assert e.value.status == 1
    with pytest.raises(ocb.B2FError) as e:
        ocb.calcOpticalFlowPyrLK(t(I0), t(I1[:50]), t(grid(60, 80)), None)
    assert e.value.status == 3
    with pytest.raises(ocb.B2FError):
        ocb.calcOpticalFlowPyrLK(t(I0), t(I1), t(grid(60, 80)), None, winSize=(2, 9))


def test_graph_capture():
    I0, I1 = frames(240, 320)
    pts = grid(240, 320, 5.0)
    lk = LK.SparsePyrLKOpticalFlow_create((11, 11), 2)
    a, b, p = t(I0), t(I1), t(pts)
    nxt = torch.empty_like(p)
    st = torch.empty((len(pts), 1), dtype=torch.uint8, device=dev)
    er = torch.zeros((len(pts), 1), dtype=torch.float32, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        lk.calc(a, b, p, nxt, st, er, stream=s)  # lays out the workspace
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        lk.calc(a, b, p, nxt, st, er, stream=s)
    nxt.zero_()
    g.replay()
    torch.cuda.synchronize()
    check((nxt, st, er), I0, I1, pts, win_size=(11, 11), max_level=2)


def test_cpp_adapter_call_site(tmp_path):
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "test_lkpyramid_compat")
    I0, I1 = frames(240, 320, shift=(3, -2))
    pts = grid(240, 320, 7.3).reshape(-1, 2)
    n = len(pts)
    for name, a in (("a", I0), ("b", I1), ("p", pts)):
        np.ascontiguousarray(a).tofile(tmp_path / name)
    out = tmp_path / "out"
    r = subprocess.run([exe, "240", "320", str(n), str(tmp_path / "a"), str(tmp_path / "b"), str(tmp_path / "p"), str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(out, np.uint8)
    assert raw.size == 4 * 13 * n
    want, st, er, wr = M.calc(I0, I1, pts, win_size=(15, 15))
    for k in range(4):
        blk = raw[k * 13 * n:(k + 1) * 13 * n]
        assert np.array_equal(blk[:8 * n].view(np.float32).reshape(-1, 2).view(np.uint32), want.view(np.uint32))
        assert np.array_equal(blk[8 * n:9 * n], st)
        assert np.array_equal(blk[9 * n:].view(np.float32)[wr & (st != 0)], er[wr & (st != 0)])


def test_pyramids_destroyed_and_recreated_between_calls():
    """One handle, pyramids freed and rebuilt (other borders, with and without derivatives) between calls: a freed
    pyramid's host address may come back for the new one, and no state of the old one may be used."""
    import gc
    I0, I1 = frames(240, 320, shift=(3, 2))
    pts = grid(240, 320, 6.3)
    tp = t(pts)
    lk = LK.SparsePyrLKOpticalFlow_create((15, 15), 3)
    for it in range(6):
        border = (15, 23, 31)[it % 3]
        m0, p0 = LK.buildOpticalFlowPyramid(t(I0), (border, border), 3, withDerivatives=it % 2 == 0)
        m1, p1 = LK.buildOpticalFlowPyramid(t(I1), (border, border), 3, withDerivatives=False)
        got = lk.calc(p0, p1, tp)
        # a 31-px border stops the pyramid at level 2 (30 rows are not larger than 31), which caps maxLevel
        assert (m0, m1) == ((2, 2) if border == 31 else (3, 3))
        check(got, I0, I1, pts, win_size=(15, 15), max_level=min(m0, m1))
        del p0, p1, got
        gc.collect()


def test_free_function_on_two_streams():
    """The top-level function's hidden handle is shared: calls on two streams must not overwrite each other's
    pyramids while a tracker still reads them."""
    A0, A1 = frames(1080, 1920, seed=11, shift=(3, 2))
    B0, B1 = frames(1080, 1920, seed=12, shift=(-2, 4))
    pa, pb = grid(1080, 1920, 9.1, 2.0), grid(1080, 1920, 9.7, 2.0)
    ta, tb = [t(x) for x in (A0, A1, pa)], [t(x) for x in (B0, B1, pb)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    outs = []
    for _ in range(3):
        with torch.cuda.stream(s1):
            ra = ocb.calcOpticalFlowPyrLK(*ta, None)
        with torch.cuda.stream(s2):
            rb = ocb.calcOpticalFlowPyrLK(*tb, None)
        outs.append((ra, rb))
    torch.cuda.synchronize()
    for ra, rb in outs:
        check(ra, A0, A1, pa, against_cv2=False)
        check(rb, B0, B1, pb, against_cv2=False)


def test_views_refuse_a_relayout_while_alive():
    import gc
    I0, _ = frames(120, 160)
    _, P = LK.buildOpticalFlowPyramid(t(I0), (9, 9), 2)
    v = P.level(0)
    LK.buildOpticalFlowPyramid(t(I0[::-1].copy()), (9, 9), 2, P)  # same geometry: allowed, the view shows the new frame
    assert np.array_equal(v.cpu().numpy().reshape(I0.shape), I0[::-1])
    with pytest.raises(ValueError):
        LK.buildOpticalFlowPyramid(t(I0[:100]), (9, 9), 2, P)
    del v
    gc.collect()
    LK.buildOpticalFlowPyramid(t(I0[:100]), (9, 9), 2, P)
    assert P.level(0).shape[:2] == (100, 160)
