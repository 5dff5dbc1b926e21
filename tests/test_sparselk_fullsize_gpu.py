"""SparsePyrLK engine against its CUDA-semantics model (oracle/sparselk_model.py), bit for bit.

The engine is built with -fmad=false, so every operator rounds once and the model follows it operator by operator.
Every comparison is np.array_equal on int32 views: nextPts over ALL points (points that returned early keep their
stale coarse estimate, which the model reproduces), status, and err wherever status is 1.  err is passed prefilled
with NaN, and the NaN must survive exactly where status is 0.  The model's per-level counters show that each input
takes the branches it is there for, and every case prints them.

Cases: the 1080p frame at create()'s defaults with border points; every entry of the reference's dispatcher table
(8U / 16U / 32S / 32F x 1 / 3 / 4 channels, both sampling paths and both kernels); windows from 3x3 to the largest the
reference accepts, including the shared-memory edges around the 48 KB default and the device's opt-in limit;
iteration counts 0 / 1 / 100; maxLevel 0 and pyramids down to 1x1; 1, 257 and 70 000 points; use_initial_flow;
pitched ROIs; one handle reused across type, size, maxLevel and window.
"""
import ctypes as C
import functools
import time

import numpy as np
import pytest

from oracle import synth, sparselk_model as sm

pytestmark = pytest.mark.gpu

B2F_BAD_ARG = 1
NP_TYPES = {"u8": np.uint8, "u16": np.uint16, "s32": np.int32, "f32": np.float32}


@functools.lru_cache(maxsize=8)
def _gray(h, w, seed, kind="const"):
    I0, I1, _ = synth.make_pair(h, w, seed=seed, kind=kind)
    return I0, I1


def _convert(a, depth):
    """Type-specific content from an 8-bit texture: u16 spans 0..65535, s32 has negative values, f32 is fractional."""
    a = a.astype(np.int64)
    if depth == "u8":
        return a.astype(np.uint8)
    if depth == "u16":
        return (a * 257).astype(np.uint16)
    if depth == "s32":
        return (a * 4099 - 500000).astype(np.int32)
    return (a.astype(np.float32) * np.float32(0.37) + np.float32(0.125)).astype(np.float32)


@functools.lru_cache(maxsize=16)
def _pair(h, w, depth="u8", cn=1, seed=3, kind="const"):
    chans = [_gray(h, w, seed + 31 * c, kind) for c in range(cn)]
    if cn == 1:
        I0, I1 = chans[0]
    else:
        I0, I1 = np.stack([c[0] for c in chans], -1), np.stack([c[1] for c in chans], -1)
    return _convert(I0, depth), _convert(I1, depth)


def _edge_points(rows, cols, half):
    """Corners, the last representable position, x = cols, x = -1e-6, points within half a window of each border and
    points near the top border, which the synthetic motion (2.5, -1.25) carries outside."""
    p = [(0, 0), (cols - 2.0 ** -8, rows - 2.0 ** -8), (cols, rows / 2), (-1e-6, rows / 2), (cols / 2, rows),
         (cols / 2, -1e-6), (0.3, 0.4), (cols - 1, rows - 1)]
    for d in (0.5, 1.0, half / 2, half - 0.5, half):
        p += [(d, rows / 2), (cols - 1 - d, rows / 2), (cols / 2, d), (cols / 2, rows - 1 - d)]
    p += [(x, y) for x in (cols * 0.3, cols * 0.7) for y in (0.25, 0.6, 1.0, 1.2)]
    return np.array(p, np.float32)


def _features(I, n, rows, cols, half, seed=0):
    gray = (I if I.ndim == 2 else I[..., 0]).astype(np.float64)
    gray = ((gray - gray.min()) / max(1e-9, float(gray.max() - gray.min())) * 255).astype(np.uint8)
    pts = cv2_features(gray, n)
    rng = np.random.default_rng(seed)
    jitter = rng.uniform(-0.5, 0.5, pts.shape).astype(np.float32)  # off the integer grid
    return np.concatenate([pts + jitter, _edge_points(rows, cols, half)]).astype(np.float32)


def cv2_features(gray, n):
    import cv2
    return cv2.goodFeaturesToTrack(gray, n, 0.01, 0.0).reshape(-1, 2).astype(np.float32)


def _run(dev, alg, I0, I1, pts, init=None, roi=0):
    """One engine call with err prefilled with NaN; returns numpy (nextPts (N, 2), status, err)."""
    import torch

    def up(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        if not roi:
            return t
        big = torch.zeros((a.shape[0], a.shape[1] + 2 * roi) + a.shape[2:], dtype=t.dtype, device=dev)
        big[:, roi:roi + a.shape[1]] = t
        view = big[:, roi:roi + a.shape[1]]
        assert view.stride(0) != a.shape[1] * (1 if a.ndim == 2 else a.shape[2])
        return view

    n = len(pts)
    p = torch.from_numpy(pts).to(dev)
    nxt = torch.from_numpy(init).to(dev) if init is not None else None
    err = torch.full((n,), float("nan"), dtype=torch.float32, device=dev)
    got, status, err = alg.calc(up(I0), up(I1), p, nxt, None, err)
    torch.cuda.synchronize()
    return got.cpu().numpy().reshape(-1, 2), status.cpu().numpy(), err.cpu().numpy()


def _model(I0, I1, pts, win, levels, iters, init=None, label=""):
    cnt = []
    t = time.perf_counter()
    want = sm.calc(I0, I1, pts, win, levels, iters, next_pts=init, counters=cnt)
    print("%s: model %.2f s, counters per level (coarsest first) %s = %s" % (
        label, time.perf_counter() - t, "/".join(sm.COUNTER_NAMES), [c.as_tuple() for c in cnt]))
    return want, cnt


def _assert_same(got, want, what):
    (gn, gs, ge), (wn, ws, we) = got, want
    bad = np.nonzero((gn.view(np.int32) != wn.view(np.int32)).any(axis=1))[0]
    if len(bad):
        i = bad[0]
        raise AssertionError("%s: nextPts of %d / %d points differ, first #%d: engine %r model %r (status %d / %d)" % (
            what, len(bad), len(gn), i, gn[i].tolist(), wn[i].tolist(), gs[i], ws[i]))
    assert np.array_equal(gs, ws), "%s: status differs at %s" % (what, np.nonzero(gs != ws)[0][:10])
    assert np.array_equal(np.isnan(ge), gs == 0), "%s: err written where status is 0, or not written where 1" % what
    ok = gs != 0
    bad = np.nonzero(ge[ok].view(np.int32) != we[ok].view(np.int32))[0]
    assert len(bad) == 0, "%s: err of %d points differs, first engine %r model %r" % (
        what, len(bad), ge[ok][bad[0]], we[ok][bad[0]])


def _compare(dev, I0, I1, pts, win=(21, 21), levels=3, iters=30, init=None, roi=0, alg=None, label=None):
    import opencv_contrib_b200 as ocb
    label = label or "%s %s win %s levels %d iters %d, %d points" % (I0.shape, I0.dtype, win, levels, iters, len(pts))
    want, cnt = _model(I0, I1, pts, win, levels, iters, init, label)
    if alg is None:
        alg = ocb.SparsePyrLKOpticalFlow_create(winSize=win, maxLevel=levels, iters=iters, useInitialFlow=init is not None)
    else:
        alg.setWinSize(win)
        alg.setMaxLevel(levels)
        alg.setNumIters(iters)
        alg.setUseInitialFlow(init is not None)
    _assert_same(_run(dev, alg, I0, I1, pts, init, roi), want, label)
    return want, cnt


def _total(cnt, name):
    return sum(getattr(c, name) for c in cnt)


def test_1080p_defaults_bit_identical_to_model(cuda_device):
    """1080x1920 8UC1 at create()'s defaults (21x21, maxLevel 3, 30 iterations), about 2 000 goodFeaturesToTrack
    points with no border mask plus the edge points."""
    I0, I1 = _pair(1080, 1920)
    pts = _features(I0, 2000, 1080, 1920, 10)
    assert len(pts) > 1900
    (_, status, _), cnt = _compare(cuda_device, I0, I1, pts)
    assert cnt[-1].outside_prev > 0 and _total(cnt, "left_during_iters") > 0 and cnt[-1].converged > 0
    assert status[-len(_edge_points(1080, 1920, 10)):].min() == 0 and status.mean() > 0.9


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("depth", ["u8", "u16", "s32", "f32"])
def test_every_dispatcher_entry_bit_identical(cuda_device, depth, cn):
    """8U / 16U / 32S / 32F with 1, 3 and 4 channels at an odd size: the texture path (8UC1, 8UC4, 16UC4, 32FC1,
    32FC4), the software path (the rest), the single-plane kernel (8UC1, 32FC1) and the multi-channel one."""
    I0, I1 = _pair(301, 403, depth, cn)
    pts = _features(I0, 300, 301, 403, 10, seed=cn)
    (_, status, _), cnt = _compare(cuda_device, I0, I1, pts)
    assert cnt[-1].outside_prev > 0 and cnt[-1].converged > 0 and status.mean() > 0.8


@pytest.mark.parametrize("win,cn", [
    ((3, 3), 1), ((4, 6), 1), ((15, 15), 1), ((16, 16), 1), ((86, 3), 1), ((21, 21), 1),
    ((80, 80), 1), ((160, 40), 1),          # the largest windows calcPatchSize accepts
    ((64, 64), 1), ((32, 32), 4), ((35, 39), 3),  # 49 152 / 49 152 / 49 140 B of patch: over 48 KB with the staging
    ((80, 80), 3), ((69, 70), 4),            # just under the H100's opt-in limit
])
def test_windows_bit_identical(cuda_device, win, cn):
    """Odd, even and asymmetric windows; fewer elements than the 256-thread block (225), exactly as many (256), more
    (258, the wide shape w > 32 && w > 2h); and the shared-memory edges."""
    I0, I1 = _pair(200, 272, "u8", cn, seed=7)
    pts = _features(I0, 40, 200, 272, max(win) // 2, seed=1)
    (_, status, _), cnt = _compare(cuda_device, I0, I1, pts, win=win, levels=2)
    assert status.any()
    if win == (64, 64):  # the same patch size on the other single-plane type
        _compare(cuda_device, I0.astype(np.float32), I1.astype(np.float32), pts, win=win, levels=2)


def test_patches_over_the_optin_limit_are_refused(cuda_device):
    """Four-channel windows whose patch does not fit in the device's opt-in shared memory are refused before any
    launch; the largest that fits runs (test_windows_bit_identical)."""
    import torch
    import opencv_contrib_b200 as ocb
    smax = torch.cuda.get_device_properties(cuda_device).shared_memory_per_block_optin
    I0, I1 = _pair(64, 96, "u8", 4)
    pts = np.array([[40.0, 30.0]], np.float32)
    for win in ((70, 70), (80, 80)):
        assert 12 * 4 * win[0] * win[1] + 96 > smax
        with pytest.raises(ocb.B2FError) as e:
            _run(cuda_device, ocb.SparsePyrLKOpticalFlow_create(winSize=win, maxLevel=1), I0, I1, pts)
        assert e.value.status == B2F_BAD_ARG
    assert 12 * 4 * 69 * 70 + 96 <= smax


@pytest.mark.parametrize("iters", [0, 1, 100])
def test_iteration_counts_bit_identical(cuda_device, iters):
    I0, I1 = _pair(240, 320, "u8", 1, seed=9, kind="affine")
    pts = _features(I0, 300, 240, 320, 10)
    _, cnt = _compare(cuda_device, I0, I1, pts, iters=iters)
    if iters == 0:
        assert all(c.converged == 0 and c.left_during_iters == 0 for c in cnt) and cnt[-1].hit_iters > 0
    elif iters == 1:
        assert cnt[-1].hit_iters > 0
    else:
        assert cnt[-1].converged > 0


@pytest.mark.parametrize("h,w,levels", [(240, 320, 0), (40, 56, 6), (40, 56, 30)])
def test_levels_bit_identical(cuda_device, h, w, levels):
    """maxLevel 0 (no pyramid); a 40x56 frame whose sixth level is 1x1; maxLevel 30, the largest accepted."""
    I0, I1 = _pair(h, w, "u8", 1, seed=13)
    pts = _features(I0, 60, h, w, 10)
    _, cnt = _compare(cuda_device, I0, I1, pts, levels=levels)
    assert len(cnt) == levels + 1


def test_max_level_over_30_is_refused(cuda_device):
    import opencv_contrib_b200 as ocb
    I0, I1 = _pair(40, 56)
    with pytest.raises(ocb.B2FError) as e:
        _run(cuda_device, ocb.SparsePyrLKOpticalFlow_create(maxLevel=31), I0, I1, np.array([[5.0, 5.0]], np.float32))
    assert e.value.status == B2F_BAD_ARG


@pytest.mark.parametrize("n", [1, 257, 70000])
def test_point_counts_bit_identical(cuda_device, n):
    I0, I1 = _pair(480, 640, "u8", 1, seed=17)
    rng = np.random.default_rng(n)
    pts = np.stack([rng.uniform(-2, 642, n), rng.uniform(-2, 482, n)], 1).astype(np.float32)
    win = (3, 3) if n > 1000 else (21, 21)
    _, cnt = _compare(cuda_device, I0, I1, pts, win=win)
    if n > 1:
        assert cnt[-1].outside_prev > 0


def test_use_initial_flow_bit_identical(cuda_device):
    """A caller estimate per point: the truth, zero motion, a wild one, and one outside the coarse level (returns early
    there and is doubled, stale, on the finer levels)."""
    I0, I1 = _pair(240, 320, "u8", 3, seed=19)
    pts = _features(I0, 200, 240, 320, 10)
    rng = np.random.default_rng(0)
    init = pts + np.float32([2.5, -1.25])
    init[::4] = pts[::4]
    init[1::4] += rng.uniform(-8, 8, init[1::4].shape).astype(np.float32)
    init[2::8] = np.float32([2000.0, 120.0])
    init = init.astype(np.float32)
    _, cnt = _compare(cuda_device, I0, I1, pts, init=init)
    assert cnt[0].left_during_iters > 0


@pytest.mark.parametrize("depth,cn", [("u8", 1), ("f32", 4), ("s32", 3)])
def test_flat_block_singular_bit_identical(cuda_device, depth, cn):
    """A flat block: points well inside it have a singular matrix (D < FLT_EPSILON) on the fine levels, not on the
    coarse ones, and keep the estimate of the last level that wrote."""
    I0, I1 = (a.copy() for a in _pair(160, 200, depth, cn, seed=31))
    I0[40:120, 50:150] = I0[0, 0]
    I1[40:120, 50:150] = I0[0, 0]
    pts = np.concatenate([_features(I0, 60, 160, 200, 10), [[100.0, 80.0], [90.5, 75.25], [110.0, 85.0]]]).astype(np.float32)
    (_, status, _), cnt = _compare(cuda_device, I0, I1, pts)
    assert cnt[-1].singular >= 3 and status[-3:].max() == 0


@pytest.mark.parametrize("depth,cn", [("u8", 1), ("u16", 4)])
def test_pitched_roi_bit_identical(cuda_device, depth, cn):
    I0, I1 = _pair(151, 203, depth, cn, seed=23)
    pts = _features(I0, 100, 151, 203, 10)
    _compare(cuda_device, I0, I1, pts, roi=5)


def test_one_handle_across_types_sizes_levels_and_windows(cuda_device):
    import opencv_contrib_b200 as ocb
    alg = ocb.SparsePyrLKOpticalFlow_create()
    for (h, w, depth, cn, win, levels) in [(120, 160, "u8", 1, (21, 21), 3), (97, 131, "u16", 4, (9, 13), 2),
                                           (120, 160, "f32", 3, (21, 21), 3), (120, 160, "u8", 1, (64, 64), 1),
                                           (60, 80, "s32", 1, (5, 5), 4), (120, 160, "u8", 1, (21, 21), 3)]:
        I0, I1 = _pair(h, w, depth, cn, seed=29)
        pts = _features(I0, 80, h, w, 10)
        _compare(cuda_device, I0, I1, pts, win=win, levels=levels, alg=alg)


def test_misaligned_pointers_are_refused(cuda_device):
    """Points are read and written as float2, 16U / 32S / 32F pixels as elements: a pointer that is not aligned to
    them is refused before any launch."""
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200 import _lib
    I0, I1 = _pair(64, 96)
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    alg = ocb.SparsePyrLKOpticalFlow_create()
    buf = torch.full((2 * 3 + 1,), 20.0, device=cuda_device)
    odd = buf[1:].view(3, 2)
    assert odd.is_contiguous() and odd.data_ptr() % 8 == 4
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(d0, d1, odd)
    assert e.value.status == B2F_BAD_ARG
    good = torch.full((3, 2), 20.0, device=cuda_device)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(d0, d1, good, torch.full((2 * 3 + 1,), 20.0, device=cuda_device)[1:].view(3, 2))
    assert e.value.status == B2F_BAD_ARG
    # a 16UC1 image whose data pointer is one byte past an element boundary
    raw = torch.zeros(64 * 192 + 2, dtype=torch.uint8, device=cuda_device)
    img = _lib.b2f_image(raw.data_ptr() + 1, 192, 64, 96, 2)
    st = torch.empty(3, dtype=torch.uint8, device=cuda_device)
    nxt = torch.empty((3, 2), device=cuda_device)
    lib = _lib.lib()
    h = alg._h
    r = lib.b2f_sparselk_calc(h, C.byref(img), C.byref(img), C.c_void_p(good.data_ptr()), C.c_void_p(nxt.data_ptr()),
                              C.c_void_p(st.data_ptr()), None, 3, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert r == B2F_BAD_ARG
    # the aligned call on the same handle still runs
    _compare(cuda_device, I0, I1, _features(I0, 20, 64, 96, 10), alg=alg)
