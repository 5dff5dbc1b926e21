"""The video module's Farneback engine (csrc/optflowgf.cu) against the live cv2 on its portable path
(setUseOptimized(False), IPP off), bit for bit on the whole flow, and against default cv2 within 4x cv2's own
default-vs-portable distance."""
import os
import subprocess

import cv2
import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import opencv_contrib_b200 as ocb  # noqa: E402
from opencv_contrib_b200 import optflowgf  # noqa: E402
from opencv_contrib_b200.batch import NativeFlowBatch  # noqa: E402

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = (0.5, 5, 13, 10, 5, 1.1, 0)


@pytest.fixture(autouse=True)
def portable():
    opt, ipp = cv2.useOptimized(), cv2.ipp.useIPP()
    cv2.setUseOptimized(False)
    cv2.ipp.setUseIPP(False)
    yield
    cv2.setUseOptimized(opt)
    cv2.ipp.setUseIPP(ipp)


def pair(rows, cols, seed=0, shift=(1, 2)):
    a = synth.texture(rows, cols, seed)
    b = np.roll(a, shift, (0, 1))
    return np.clip(np.rint(a), 0, 255).astype(np.uint8), np.clip(np.rint(b), 0, 255).astype(np.uint8)


def neq(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape
    return int((a.view(np.uint32) != b.view(np.uint32)).sum())


def cv_flow(a, b, flow, args):
    return cv2.calcOpticalFlowFarneback(a, b, None if flow is None else flow.copy(), *args)


def gpu_flow(a, b, flow, args, stream=None):
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    df = None if flow is None else torch.from_numpy(flow.copy()).cuda()
    out = ocb.calcOpticalFlowFarneback(da, db, df, *args, stream=stream)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def check(a, b, flow, args):
    assert neq(cv_flow(a, b, flow, args), gpu_flow(a, b, flow, args)) == 0


@pytest.mark.parametrize("shape", [(1, 1), (1, 37), (37, 1), (3, 4), (9, 12), (31, 31), (32, 32), (33, 33), (63, 64),
                                   (64, 65), (65, 63), (12, 200), (97, 131)])
def test_sizes(shape):
    a, b = pair(*shape)
    check(a, b, None, BASE)
    check(a, b, None, (0.5, 5, 13, 3, 5, 1.1, 256))


@pytest.mark.parametrize("args", [
    (0.8, 5, 13, 3, 5, 1.1, 0), (0.3, 5, 13, 3, 5, 1.1, 0), (0.0, 5, 13, 3, 5, 1.1, 0), (-0.5, 3, 13, 2, 5, 1.1, 0),
    (0.5, 0, 13, 3, 5, 1.1, 0), (0.5, 1, 13, 3, 5, 1.1, 0), (0.5, 3, 13, 3, 5, 1.1, 0), (0.5, -2, 13, 3, 5, 1.1, 0),
    (0.5, 5, 1, 3, 5, 1.1, 0), (0.5, 5, 2, 3, 5, 1.1, 0), (0.5, 5, 14, 3, 5, 1.1, 0), (0.5, 5, 31, 3, 5, 1.1, 0),
    (0.5, 5, 13, 0, 5, 1.1, 0), (0.5, 5, 13, 1, 5, 1.1, 0), (0.5, 5, 13, 2, 5, 1.1, 0), (0.5, 5, 13, 10, 5, 1.1, 0),
    (0.5, 5, 13, 3, 7, 1.5, 0), (0.5, 5, 13, 3, 3, 1.1, 0), (0.5, 5, 13, 3, 6, 1.3, 0), (0.5, 5, 13, 3, 5, 0.0, 0),
    (0.5, 5, 1, 3, 5, 1.1, 256), (0.5, 5, 2, 3, 5, 1.1, 256), (0.5, 5, 14, 3, 7, 1.5, 256), (0.5, 5, 31, 2, 5, 1.1, 256),
    (0.8, 5, 5, 10, 6, 0.0, 256), (0.5, 5, 13, 3, 15, 3.0, 0)])
def test_parameters(args):
    a, b = pair(97, 131, seed=3, shift=(2, -3))
    check(a, b, None, args)


@pytest.mark.parametrize("rows", [30, 63, 64, 65, 129])
@pytest.mark.parametrize("flags", [0, 256])
@pytest.mark.parametrize("iters", [2, 3])
def test_heights(rows, flags, iters):
    a, b = pair(rows, 40, seed=rows)
    check(a, b, None, (0.5, 0, 5, iters, 5, 1.1, flags))


def initial_flows(rows, cols):
    ys, xs = np.mgrid[0:rows, 0:cols].astype(np.float32)
    return {"zero": np.zeros((rows, cols, 2), np.float32),
            "smooth": synth.flow_field(rows, cols, "smooth", seed=1, mag=4.0),
            "huge": np.full((rows, cols, 2), 1e4, np.float32),
            "out": np.stack([-xs - 5, (rows - ys) + 3], -1).astype(np.float32),
            "neg_zero": np.full((rows, cols, 2), -0.0, np.float32)}


@pytest.mark.parametrize("kind", ["zero", "smooth", "huge", "out", "neg_zero"])
@pytest.mark.parametrize("flags", [4, 4 | 256])
@pytest.mark.parametrize("shape,levels", [((97, 131), 5), ((128, 160), 5), ((97, 131), 0), ((120, 150), 2)])
def test_initial_flow(kind, flags, shape, levels):
    a, b = pair(*shape, seed=5)
    check(a, b, initial_flows(*shape)[kind], (0.5, levels, 9, 2, 5, 1.1, flags))


def test_initial_flow_pyr_scale_08():
    a, b = pair(100, 140, seed=6)
    check(a, b, initial_flows(100, 140)["smooth"], (0.8, 5, 9, 2, 5, 1.1, 4))


def test_handle_changes_window_and_initial_flow():
    """one handle: box, gaussian, initial flow and back; the workspace is re-laid out for each"""
    a, b = pair(97, 131, seed=60)
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    fb = optflowgf.FarnebackOpticalFlow_create()
    init = initial_flows(97, 131)["smooth"]
    for flags in (0, 256, 4, 4 | 256, 0):
        fb.setFlags(flags)
        f = torch.from_numpy(init.copy()).cuda() if flags & 4 else None
        out = fb.calc(da, db, f)
        torch.cuda.synchronize()
        assert neq(cv_flow(a, b, init if flags & 4 else None, BASE[:6] + (flags,)), out.cpu().numpy()) == 0


@pytest.mark.parametrize("shape", [(480, 640), (1080, 1920)])
@pytest.mark.parametrize("flags", [0, 256, 4, 4 | 256])
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_benchmark_sizes(shape, flags, dtype):
    a, b = synth.make_pair(*shape, seed=0, kind="smooth")[:2]
    a, b = np.clip(np.rint(a), 0, 255).astype(dtype), np.clip(np.rint(b), 0, 255).astype(dtype)
    if dtype == np.float32:
        a = a * np.float32(1.7) - np.float32(40.25)
        b = b * np.float32(1.7) - np.float32(40.25)
    flow = synth.flow_field(*shape, "smooth", seed=2, mag=3.0) if flags & 4 else None
    check(a, b, flow, BASE[:6] + (flags,))


def test_pitched_roi_frames_and_flow():
    a, b = pair(101, 133, seed=11)
    da = torch.zeros((101, 160), dtype=torch.uint8, device="cuda")
    db = torch.zeros((101, 192), dtype=torch.uint8, device="cuda")
    da[:, 3:136] = torch.from_numpy(a).cuda()
    db[:, 17:150] = torch.from_numpy(b).cuda()
    init = synth.flow_field(101, 133, "smooth", seed=3, mag=2.0)
    fbuf = torch.full((101, 150, 2), 7.0, device="cuda")
    fbuf[:, 5:138] = torch.from_numpy(init).cuda()
    args = (0.5, 5, 9, 3, 5, 1.1, 4)
    out = ocb.calcOpticalFlowFarneback(da[:, 3:136], db[:, 17:150], fbuf[:, 5:138], *args)
    torch.cuda.synchronize()
    assert neq(cv_flow(a, b, init, args), out.cpu().numpy()) == 0
    assert bool((fbuf[:, :5] == 7).all()) and bool((fbuf[:, 138:] == 7).all())


def test_calc_uv_calc_host_and_class():
    a, b = pair(97, 131, seed=12)
    ref = cv_flow(a, b, None, BASE)
    fb = optflowgf.FarnebackOpticalFlow_create(5, 0.5, True, 13, 10, 5, 1.1, 0)
    assert fb.getDefaultName() == "DenseOpticalFlow.FarnebackOpticalFlow"
    assert fb.getFastPyramids() is True and fb.getWinSize() == 13 and fb.getPolySigma() == 1.1
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    u, v = fb.calcUV(da, db)
    torch.cuda.synchronize()
    assert neq(ref, np.stack([u.cpu().numpy(), v.cpu().numpy()], -1)) == 0
    assert neq(ref, fb.calc_host(a, b)) == 0
    assert fb.getActivePath(0) == optflowgf.PATH["box"]
    fb.setFlags(256)
    fb.calc(da, db)
    assert fb.getActivePath(0) & optflowgf.PATH["gaussian"]


def test_refusals():
    a = torch.zeros((40, 40), dtype=torch.uint8, device="cuda")
    for kw in [dict(polyN=16), dict(polyN=0), dict(winSize=0), dict(winSize=256), dict(pyrScale=1.0)]:
        with pytest.raises(ocb.B2FError):
            optflowgf.FarnebackOpticalFlow_create(**kw).calc(a, a)
    with pytest.raises(ocb.B2FError):
        optflowgf.FarnebackOpticalFlow_create().calc(a.to(torch.int16), a.to(torch.int16))


def test_batch_algo_9():
    pairs = [pair(120, 160, seed=s, shift=(s % 3, 2)) for s in range(6)]
    nb = NativeFlowBatch("optflowgf", dict(win_size=9, flags=256), n_streams=3)
    I0 = [torch.from_numpy(p[0]).cuda() for p in pairs]
    I1 = [torch.from_numpy(p[1]).cuda() for p in pairs]
    flows = [torch.empty((120, 160, 2), dtype=torch.float32, device="cuda") for _ in pairs]
    nb.run_device(list(zip(I0, I1)), flows)
    torch.cuda.synchronize()
    for (a, b), f in zip(pairs, flows):
        assert neq(cv_flow(a, b, None, (0.5, 5, 9, 10, 5, 1.1, 256)), f.cpu().numpy()) == 0
    nb.close()


def test_video_warm_start_equals_pairwise():
    frames = [np.clip(np.rint(synth.texture(96, 128, 0)), 0, 255).astype(np.uint8)]
    for k in range(4):
        frames.append(np.roll(frames[0], (k + 1, 2 * (k + 1)), (0, 1)))
    fb = optflowgf.FarnebackOpticalFlow_create(numIters=3)
    vid = ocb.VideoFlow(fb, 96, 128, depth=2, warm_start=True)
    got = [f.copy() for _, f in vid.run(frames)]
    prev = None
    for k in range(4):
        args = (0.5, 5, 13, 3, 5, 1.1, 0 if prev is None else 4)
        prev = cv_flow(frames[k], frames[k + 1], prev, args)
        assert neq(prev, got[k]) == 0
    vid.close()


def test_four_handles_on_four_streams():
    pairs = [pair(150, 200, seed=20 + i) for i in range(4)]
    streams = [torch.cuda.Stream() for _ in range(4)]
    handles = [optflowgf.FarnebackOpticalFlow_create(flags=256 * (i % 2)) for i in range(4)]
    dev = [(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) for a, b in pairs]
    torch.cuda.synchronize()
    outs = []
    for rep in range(3):
        for i in range(4):
            with torch.cuda.stream(streams[i]):
                outs.append((i, handles[i].calc(*dev[i], stream=streams[i])))
    torch.cuda.synchronize()
    for i, o in outs:
        ref = cv_flow(*pairs[i], None, (0.5, 5, 13, 10, 5, 1.1, 256 * (i % 2)))
        assert neq(ref, o.cpu().numpy()) == 0


def test_graph_replay_and_recapture():
    a, b = pair(120, 160, seed=30)
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    s = torch.cuda.Stream()
    fb = optflowgf.FarnebackOpticalFlow_create()
    for args, setter in [(BASE, None), (BASE, None), ((0.5, 5, 9, 10, 5, 1.1, 0), ("setWinSize", 9)),
                         ((0.5, 5, 9, 10, 7, 1.5, 0), ("setPolyN", 7)), ((0.5, 5, 9, 10, 7, 1.5, 0), None)]:
        if setter:
            getattr(fb, setter[0])(setter[1])
        if setter and setter[0] == "setPolyN":
            fb.setPolySigma(1.5)
        out = fb.calc(da, db, stream=s)
        s.synchronize()
        assert neq(cv_flow(a, b, None, args), out.cpu().numpy()) == 0


def test_cpp_adapter_two_streams():
    """the C++ free function on two non-blocking streams back to back, and the C++ class, against cv2"""
    exe = os.path.join(_ROOT, "tests", "cpp", "test_optflowgf_compat")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    hexes = r.stdout.split()[-2:]
    frames = [np.fromfunction(lambda y, x, k=k: ((x * 7 + y * 3 + k * 5) % 64) * 4, (64, 80)).astype(np.uint8)
              for k in range(3)]
    for k, hx in zip((1, 2), hexes):
        got = np.frombuffer(bytes.fromhex(hx), np.float32).reshape(64, 80, 2)
        assert neq(cv_flow(frames[0], frames[k], None, (0.5, 3, 9, 3, 5, 1.1, 0)), got) == 0


def test_free_function_on_two_streams():
    """one thread, one handle, two streams, no synchronisation between the calls"""
    (a, b), (c, d) = pair(240, 320, seed=40), pair(240, 320, seed=41, shift=(3, -1))
    dev = [torch.from_numpy(x).cuda() for x in (a, b, c, d)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(3):
        f1 = ocb.calcOpticalFlowFarneback(dev[0], dev[1], None, *BASE, stream=s1)
        f2 = ocb.calcOpticalFlowFarneback(dev[2], dev[3], None, 0.5, 5, 13, 10, 5, 1.1, 256, stream=s2)
    torch.cuda.synchronize()
    assert neq(cv_flow(a, b, None, BASE), f1.cpu().numpy()) == 0
    assert neq(cv_flow(c, d, None, (0.5, 5, 13, 10, 5, 1.1, 256)), f2.cpu().numpy()) == 0


def test_deepest_blur_refusal():
    """at pyrScale 0.5 a shorter side of 4096 with 7 levels reaches 1/scale 128: ksize 319 > 255 is refused; 6 levels
    (ksize 159) are not"""
    img = torch.zeros((4096, 4096), dtype=torch.uint8, device="cuda")
    with pytest.raises(ocb.B2FError):
        optflowgf.FarnebackOpticalFlow_create(numLevels=7, numIters=1).calc(img, img)
    narrow = torch.zeros((4096, 4095), dtype=torch.uint8, device="cuda")
    fb = optflowgf.FarnebackOpticalFlow_create(numLevels=7, numIters=1)
    fb.calc(narrow, narrow)  # 4095 / 128 < 32: six levels
    torch.cuda.synchronize()
    assert fb.getStats()["levels"] == 7


def test_area_level_path_bit():
    """640x480 at pyrScale 0.5: level 1 (320x240) is an exact half, resized by the fast-area rule; the others are not"""
    a, b = pair(480, 640, seed=50)
    fb = optflowgf.FarnebackOpticalFlow_create(numIters=1)
    fb.calc(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda())
    torch.cuda.synchronize()
    bits = [fb.getActivePath(lv) & optflowgf.PATH["area_level"] for lv in range(4)]
    assert bits == [0, optflowgf.PATH["area_level"], 0, 0]


@pytest.mark.parametrize("flags", [0, 256])
def test_close_to_default_cv2(flags):
    a, b = synth.make_pair(480, 640, seed=0, kind="smooth")[:2]
    a, b = np.clip(np.rint(a), 0, 255).astype(np.uint8), np.clip(np.rint(b), 0, 255).astype(np.uint8)
    args = BASE[:6] + (flags,)
    ours = gpu_flow(a, b, None, args)
    port = cv_flow(a, b, None, args)
    cv2.setUseOptimized(True)
    cv2.ipp.setUseIPP(True)
    dflt = cv_flow(a, b, None, args)
    d_ours = np.linalg.norm(dflt - ours, axis=-1)
    d_cv = np.linalg.norm(dflt - port, axis=-1)
    assert d_ours.mean() <= 4 * d_cv.mean() + 1e-12
    assert d_ours.max() <= 4 * d_cv.max() + 1e-12
