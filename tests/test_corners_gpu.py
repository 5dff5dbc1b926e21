"""GPU tests for cudaimgproc's corner classes: the response kernel and the GoodFeaturesToTrack detector equal
oracle/corners_model.py bit for bit (same N, same coordinates, same order), and the detector feeds SparsePyrLK on the
device.  The end-to-end check against the live CPU cv2.goodFeaturesToTrack uses the reference test's criterion
(modules/cudaimgproc/test/test_gftt.cpp): the same count and at most 1 % of the points at another position."""
import ctypes as C
import threading

import cv2
import numpy as np
import pytest

from oracle import corners_model as M
from oracle import synth

pytestmark = pytest.mark.gpu


def _img(rows, cols, seed=0, f32=False):
    a = np.clip(np.rint(synth.texture(rows, cols, seed)), 0, 255).astype(np.uint8)
    return (a / np.float32(255)).astype(np.float32) if f32 else a


def _t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _criterion(harris, f32, bs, ks, border):
    import opencv_contrib_b200 as ocb
    t = 5 if f32 else 0
    return ocb.createHarrisCorner(t, bs, ks, 0.04, border) if harris else ocb.createMinEigenValCorner(t, bs, ks, border)


@pytest.mark.parametrize("harris", [False, True])
@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("ks", [-1, 0, 1, 3, 5, 7])
@pytest.mark.parametrize("border", [4, 1, 2])
def test_response_equals_model_every_aperture_border_depth(cuda_device, harris, f32, ks, border):
    src = _img(480, 640, seed=1, f32=f32)
    for bs in (1, 2, 3, 4, 5, 7):
        got = _criterion(harris, f32, bs, ks, border).compute(_t(src, cuda_device)).cpu().numpy()
        want = M.response(src, bs, ks, border, harris)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (bs, np.abs(got - want).max())


@pytest.mark.parametrize("shape", [(1080, 1920), (15, 31), (17, 33), (16, 32), (31, 63), (33, 65), (47, 97), (49, 95),
                                   (1, 40), (40, 1), (1, 1), (2, 3), (5, 4), (64, 1)])
def test_response_equals_model_at_tile_edge_and_tiny_shapes(cuda_device, shape):
    for harris, f32, bs, ks, border in ((False, False, 3, 3, 4), (True, True, 7, 5, 2), (False, True, 31, 7, 1),
                                        (True, False, 5, 0, 4), (False, False, 30, 3, 4), (True, True, 6, 1, 1)):
        src = _img(*shape, seed=2, f32=f32)
        got = _criterion(harris, f32, bs, ks, border).compute(_t(src, cuda_device)).cpu().numpy()
        want = M.response(src, bs, ks, border, harris)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (harris, f32, bs, ks, border)


def test_response_on_a_pitched_roi(cuda_device):
    big = _img(300, 400, seed=3)
    src = _t(big, cuda_device)[17:217, 33:333]
    dst = _t(np.zeros((260, 512), np.float32), cuda_device)[5:205, 7:307]
    _criterion(False, False, 5, 3, 4).compute(src, dst)
    want = M.response(np.ascontiguousarray(big[17:217, 33:333]), 5, 3, 4, False)
    assert np.array_equal(dst.cpu().numpy(), want)


def _detect(det, img, dev, mask=None):
    out = det.detect(_t(img, dev), _t(mask, dev) if mask is not None else None)
    return out.cpu().numpy().reshape(-1, 2)


@pytest.mark.parametrize("md", [0.0, 1.0, 2.4, 3.0, 10.0])
@pytest.mark.parametrize("mc", [0, 1, 1000])
@pytest.mark.parametrize("harris", [False, True])
def test_detect_equals_model(cuda_device, md, mc, harris):
    import opencv_contrib_b200 as ocb
    img = _img(240, 320, seed=4)
    mask = np.zeros_like(img)
    mask[20:200, 30:290] = 1
    det = ocb.createGoodFeaturesToTrackDetector(0, mc, 0.01, md, 3, harris, 0.04)
    for m in (None, mask):
        got = _detect(det, img, cuda_device, m)
        want, _ = M.gftt(img, mc, 0.01, md, 3, harris, 0.04, m)
        assert got.shape == want.shape and np.array_equal(got, want), (m is None, got.shape, want.shape)
        if md >= 1:
            kept, _ = M.candidates(M.response(img, 3, 3, M.BORDER_REFLECT101, harris, 0.04), 0.01, m)
            assert det.lastInfo()["rounds"] == M.selection_rounds(kept, md, 240, 320)


def test_flat_image_gives_an_empty_result(cuda_device):
    import opencv_contrib_b200 as ocb
    det = ocb.createGoodFeaturesToTrackDetector(0)
    out = det.detect(_t(np.full((64, 80), 7, np.uint8), cuda_device))
    assert tuple(out.shape) == (1, 0, 2)


def _tie_image():
    img = np.zeros((96, 128), np.uint8)
    for y in range(8, 88, 8):
        for x in range(8, 120, 8):
            img[y:y + 3, x:x + 3] = 200  # identical blobs: equal responses, more than 3 px apart
    return img


@pytest.mark.parametrize("md", [0.0, 3.0, 9.0])
def test_tie_heavy_image(cuda_device, md):
    import opencv_contrib_b200 as ocb
    img = _tie_image()
    det = ocb.createGoodFeaturesToTrackDetector(0, 50, 0.01, md)
    got = _detect(det, img, cuda_device)
    want, _ = M.gftt(img, 50, 0.01, md)
    assert len(want) > 10 and np.array_equal(got, want)


def test_capacity_cut_is_deterministic(cuda_device):
    import opencv_contrib_b200 as ocb
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (200, 200), dtype=np.uint8)  # noise: far more local maxima than max(1000, 5 %)
    for md in (0.0, 2.0):
        det = ocb.createGoodFeaturesToTrackDetector(0, 0, 0.001, md)
        want, n = M.gftt(img, 0, 0.001, md)
        first = None
        for _ in range(3):
            got = _detect(det, img, cuda_device)
            info = det.lastInfo()
            assert info["capped"] and info["candidates"] == n > info["kept"] == M.keep_capacity(200, 200)
            assert np.array_equal(got, want)
            if first is not None:
                assert np.array_equal(first, got)
            first = got


def test_selection_runs_many_rounds(cuda_device):
    import opencv_contrib_b200 as ocb
    # a diagonal ramp of isolated peaks, strongest at the top left: each peak's candidate conflicts with the next one,
    # so each decision waits for the one before it -- one round per link of the chain
    img = np.zeros((128, 128), np.float32)
    for i in range(40):
        img[3 + 3 * i, 3 + 3 * i] = 1.0 - i * 0.01
    det = ocb.createGoodFeaturesToTrackDetector(5, 0, 0.001, 5.0)
    got = _detect(det, img, cuda_device)
    info = det.lastInfo()
    want, _ = M.gftt(img, 0, 0.001, 5.0)
    kept, _ = M.candidates(M.response(img, 3, 3), 0.001)
    assert np.array_equal(got, want)
    assert info["rounds"] == M.selection_rounds(kept, 5.0, 128, 128) == 40, info


def test_detect_and_compute_are_graph_capturable(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    img = _t(_img(240, 320, seed=6), cuda_device)
    det = ocb.createGoodFeaturesToTrackDetector(0, 500, 0.01, 3.0)
    crit = ocb.createMinEigenValCorner(0, 3, 3)
    s = torch.cuda.Stream(cuda_device)
    with torch.cuda.stream(s):
        det.detect_async(img, stream=s)  # lays out the workspace: a capture cannot allocate
        eig = torch.zeros((240, 320), dtype=torch.float32, device=cuda_device)
        corners = torch.zeros((det.capacity(240, 320), 2), dtype=torch.float32, device=cuda_device)
        count = torch.zeros((1,), dtype=torch.int32, device=cuda_device)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        det.detect_async(img, corners=corners, count=count, stream=s)
        crit.compute(img, eig, stream=s)
    want, _ = M.gftt(img.cpu().numpy(), 500, 0.01, 3.0)
    for _ in range(2):
        corners.zero_()
        count.zero_()
        eig.zero_()
        g.replay()
        torch.cuda.synchronize()
        n = int(count.item())
        assert n == len(want) and np.array_equal(corners[:n].cpu().numpy(), want)
        assert np.array_equal(eig.cpu().numpy(), M.response(img.cpu().numpy(), 3, 3))
    # a detect on a size the workspace is not laid out for is refused inside a capture, before any launch
    other = _t(_img(100, 120, seed=6), cuda_device)
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(ocb.B2FError):
        with torch.cuda.graph(g2, stream=s):
            det.detect_async(other, corners=corners, count=count, stream=s)


def test_detect_then_track_on_the_device(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(360, 480, seed=21, kind="const")
    mask = np.zeros_like(I0)
    mask[12:-12, 12:-12] = 255
    det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, 0.0)
    d0, d1 = _t(I0, cuda_device), _t(I1, cuda_device)
    pts = det.detect(d0, _t(mask, cuda_device))
    lk = ocb.SparsePyrLKOpticalFlow_create()
    nxt, st, _ = lk.calc(d0, d1, pts)
    want, _ = M.gftt(I0, 1000, 0.01, 0.0, mask=mask)
    nxt2, st2, _ = lk.calc(d0, d1, torch.from_numpy(want).to(cuda_device).reshape(1, -1, 2))
    assert np.array_equal(nxt.cpu().numpy(), nxt2.cpu().numpy()) and np.array_equal(st.cpu().numpy(), st2.cpu().numpy())


@pytest.mark.parametrize("md", [0.0, 3.0])
def test_against_live_cpu_reference_at_1080p(cuda_device, md):
    import opencv_contrib_b200 as ocb
    img = _img(1080, 1920, seed=7)
    det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, md)
    got = _detect(det, img, cuda_device)
    cpu = cv2.goodFeaturesToTrack(img, 1000, 0.01, md).reshape(-1, 2)
    assert len(got) == len(cpu)
    bad = np.mean(np.any(got.astype(np.int32) != cpu.astype(np.int32), axis=1))
    assert bad <= 0.01, bad


def test_bad_arguments_are_refused(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200 import _lib
    l = _lib.lib()
    h = C.c_void_p()
    assert l.b2f_harris_create(0, 3, 3, 0.04, 0, C.byref(h)) == 1       # BORDER_CONSTANT
    assert l.b2f_harris_create(0, 3, 2, 0.04, 4, C.byref(h)) == 1       # even aperture
    assert l.b2f_mineig_create(0, 0, 3, 4, C.byref(h)) == 1             # blockSize 0
    assert l.b2f_mineig_create(0, 32, 3, 4, C.byref(h)) == 1            # above 31
    assert l.b2f_mineig_create(2, 3, 3, 4, C.byref(h)) == 2             # 16U
    for kw in (dict(qualityLevel=0.0), dict(minDistance=-1.0), dict(maxCorners=-1)):
        with pytest.raises(ocb.B2FError):
            ocb.createGoodFeaturesToTrackDetector(0, **kw)
    det = ocb.createGoodFeaturesToTrackDetector(0)
    img = _t(_img(64, 64), cuda_device)
    with pytest.raises(ocb.B2FError):
        det.detect(img.float())                                             # type differs from srcType
    with pytest.raises(ocb.B2FError):
        det.detect(img, torch.zeros((64, 63), dtype=torch.uint8, device=cuda_device))  # mask size
    small = torch.zeros((10, 2), dtype=torch.float32, device=cuda_device)
    with pytest.raises(ocb.B2FError):
        det.detect_async(img, corners=small)                                # below b2f_gftt_capacity
    crit = ocb.createMinEigenValCorner(0, 3, 3)
    with pytest.raises(ocb.B2FError):
        crit.compute(img, torch.zeros((64, 65), dtype=torch.float32, device=cuda_device))


def test_two_detectors_two_streams_two_threads(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    imgs = [_t(_img(480, 640, seed=s), cuda_device) for s in (8, 9)]
    want = [M.gftt(i.cpu().numpy(), 1000, 0.01, 3.0)[0] for i in imgs]
    out = [None, None]

    def run(k):
        det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, 3.0)
        s = torch.cuda.Stream(cuda_device)
        res = []
        for _ in range(5):
            res.append(det.detect(imgs[k], stream=s).cpu().numpy().reshape(-1, 2))
        out[k] = res

    th = [threading.Thread(target=run, args=(k,)) for k in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for k in (0, 1):
        assert all(np.array_equal(r, want[k]) for r in out[k])
