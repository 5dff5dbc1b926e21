"""BTV-L1 super-resolution on the GPU (b2f_superres_*, b2f_calc_ext) against its float model, oracle/superres_model:
the float output with ==, the 8-bit output with ==."""
import ctypes as C

import cv2
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import opencv_contrib_b200 as ocb  # noqa: E402
from opencv_contrib_b200 import _lib, superres  # noqa: E402
from oracle import superres_model as M  # noqa: E402

DEV = torch.device("cuda:0")


def _frames(n, h, w, cn, seed):
    rng = np.random.default_rng(seed)
    base = cv2.resize(rng.integers(0, 256, (h // 2 + 3, w // 2 + 3, cn), dtype=np.uint8), (w + 6, h + 6),
                      interpolation=cv2.INTER_CUBIC).reshape(h + 6, w + 6, cn)
    out = []
    for t in range(n):
        f = base[t % 3:t % 3 + h, (2 * t) % 5:(2 * t) % 5 + w]
        noise = rng.integers(-20, 21, f.shape)
        f = np.clip(f.astype(int) + noise, 0, 255).astype(np.uint8)
        out.append(f[..., 0] if cn == 1 else np.ascontiguousarray(f))
    return out


def _flows(n, h, w, seed, lo=-2.0, hi=2.0):
    rng = np.random.default_rng(seed)
    return [(rng.uniform(lo, hi, (h, w)).astype(np.float32), rng.uniform(lo, hi, (h, w)).astype(np.float32))
            for _ in range(2 * max(n - 1, 0))]


class ListFlow:
    """A caller-supplied flow object (the reference perf test's ZeroOpticalFlow pattern): hands out precomputed flows in
    the order the schedule asks for them."""

    def __init__(self, flows):
        self.flows, self.i = flows, 0

    def calc(self, f0, f1, u, v):
        a, b = self.flows[self.i]
        self.i += 1
        return torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)


def _engine(frames, flow_obj, P, float_output=True, **opts):
    sr = ocb.createSuperResolution_BTVL1_CUDA()
    sr.setOpticalFlow(flow_obj)
    for name, v in (("Scale", P.scale), ("Iterations", P.iterations), ("Tau", P.tau), ("Lambda", P.lambda_),
                    ("Alpha", P.alpha), ("KernelSize", P.btv_kernel_size), ("BlurKernelSize", P.blur_kernel_size),
                    ("BlurSigma", P.blur_sigma), ("TemporalAreaRadius", P.temporal_area_radius)):
        getattr(sr, "set" + name)(v)
    for k, v in opts.items():
        sr.setEngineOption(k, v)
    sr.setInput(frames)
    outs = []
    while (o := sr.nextFrame(float_output=float_output)) is not None:
        outs.append(o.cpu().numpy())
    return outs, sr


def _model(frames, flows, P):
    it = iter(flows)
    outs, _ = M.run(frames, lambda a, b: next(it), P)
    return outs


def _check(frames, flows, P):
    want = _model(frames, flows, P)
    got, _ = _engine(frames, ListFlow(flows), P)
    assert len(got) == len(want) == len(frames)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g, w), (i, np.abs(g - w).max())
    got8, _ = _engine(frames, ListFlow(flows), P, float_output=False)
    for g, w in zip(got8, want):
        assert np.array_equal(g, M.to_u8(w))


@pytest.mark.parametrize("cn", [1, 3, 4])
@pytest.mark.parametrize("scale", [2, 3, 4])
def test_channels_and_scales(cn, scale):
    n, h, w = 4, 11, 14
    P = M.Params(scale=scale, iterations=4, temporal_area_radius=1, btv_kernel_size=5)
    _check(_frames(n, h, w, cn, seed=cn * 10 + scale), _flows(n, h, w, seed=scale), P)


@pytest.mark.parametrize("btv", [1, 3, 7, 16])
def test_btv_kernel_sizes(btv):
    n, h, w = 3, 18, 20
    P = M.Params(scale=2, iterations=3, temporal_area_radius=1, btv_kernel_size=btv)
    _check(_frames(n, h, w, 3, seed=btv), _flows(n, h, w, seed=btv), P)


@pytest.mark.parametrize("blur,sigma", [(1, 0.0), (5, 0.0), (7, 0.0), (5, 1.3), (7, 1.3), (31, 0.0)])
@pytest.mark.parametrize("lam", [0.0, 0.03])
def test_blur_and_lambda(blur, sigma, lam):
    n, h, w = 3, 10, 13
    P = M.Params(scale=2, iterations=3, temporal_area_radius=1, blur_kernel_size=blur, blur_sigma=sigma, lambda_=lam)
    _check(_frames(n, h, w, 1, seed=blur), _flows(n, h, w, seed=blur + 1), P)


@pytest.mark.parametrize("R", [0, 1, 4])
@pytest.mark.parametrize("n", [1, 2, 5, 11])
def test_radius_and_stream_lengths(R, n):
    h, w = 9, 12
    P = M.Params(scale=2, iterations=2, temporal_area_radius=R, btv_kernel_size=3)
    _check(_frames(n, h, w, 3, seed=R * 7 + n), _flows(n, h, w, seed=n), P)


def test_flows_past_every_border():
    """Flows that push the maps far outside the image, into (-1, 0), and to huge values."""
    n, h, w = 4, 10, 12
    flows = _flows(n, h, w, seed=3, lo=-30.0, hi=30.0)
    flows[0] = (np.full((h, w), -0.3, np.float32), np.full((h, w), -0.45, np.float32))
    flows[1] = (np.full((h, w), 1e9, np.float32), np.full((h, w), -1e9, np.float32))
    P = M.Params(scale=4, iterations=3, temporal_area_radius=2)
    _check(_frames(n, h, w, 1, seed=3), flows, P)


def test_wrappers_equal_cvtcolor_then_engine():
    f0, f1 = _frames(2, 40, 48, 3, seed=5)
    g0, g1 = cv2.cvtColor(f0, cv2.COLOR_BGR2GRAY), cv2.cvtColor(f1, cv2.COLOR_BGR2GRAY)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    for make, engine, to_f32 in ((ocb.createOptFlow_Farneback_CUDA, ocb.FarnebackOpticalFlow_create(), False),
                                 (ocb.createOptFlow_DualTVL1_CUDA, ocb.OpticalFlowDual_TVL1_create(), False),
                                 (ocb.createOptFlow_PyrLK_CUDA, ocb.DensePyrLKOpticalFlow_create(), False)):
        u, v = make().calc(t(f0), t(f1), None, True)
        wu, wv = engine.calcUV(t(g0), t(g1))
        assert torch.equal(u, wu) and torch.equal(v, wv), make.__name__
    bgra = np.concatenate([f0, np.full(f0.shape[:2] + (1,), 9, np.uint8)], -1)
    bgra1 = np.concatenate([f1, np.full(f1.shape[:2] + (1,), 200, np.uint8)], -1)
    brox = ocb.createOptFlow_Brox_CUDA()
    brox.setOuterIterations(3)
    flow = brox.calc(t(bgra), t(bgra1))
    e = ocb.BroxOpticalFlow_create(float(np.float32(0.197)), float(np.float32(50.0)), float(np.float32(0.8)), 10, 3, 10)
    want = e.calc(t(M.gray(bgra, True)), t(M.gray(bgra1, True)))
    assert torch.equal(flow, want)
    assert brox.getOuterIterations() == 3 and brox.getInnerIterations() == 10


@pytest.mark.parametrize("make", ["createOptFlow_Farneback_CUDA", "createOptFlow_DualTVL1_CUDA",
                                  "createOptFlow_Brox_CUDA", "createOptFlow_PyrLK_CUDA"])
def test_superres_on_each_wrapper_equals_model_on_its_flows(make):
    n, h, w = 3, 24, 32
    frames = _frames(n, h, w, 3, seed=11)
    wrapper = getattr(ocb, make)()
    if make == "createOptFlow_Brox_CUDA":
        wrapper.setOuterIterations(4)
    if make == "createOptFlow_DualTVL1_CUDA":
        wrapper.setIterations(20)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    flows = []
    for i in range(n - 1):
        for a, b in ((frames[i], frames[i + 1]), (frames[i + 1], frames[i])):
            u, v = wrapper.calc(t(a), t(b), None, True)
            flows.append((u.cpu().numpy(), v.cpu().numpy()))
    P = M.Params(scale=2, iterations=3, temporal_area_radius=1)
    want = _model(frames, flows, P)
    got, sr = _engine(frames, wrapper, P)
    assert len(got) == n
    for g, wv in zip(got, want):
        assert np.array_equal(g, wv)


def test_reference_perf_config_and_large_output():
    # perf_superres.cpp:118-152: 128 x 128, scale 2, 50 iterations, R = 1, zero flow, the same frame every call
    frame = _frames(1, 128, 128, 1, seed=1)[0]
    n = 4
    zero = [(np.zeros((128, 128), np.float32),) * 2] * (2 * (n - 1))
    P = M.Params(scale=2, iterations=50, temporal_area_radius=1)
    _check([frame] * n, zero, P)
    # 240 x 135 x 3 -> 960 x 540 at scale 4
    frames = _frames(3, 135, 240, 3, seed=2)
    P = M.Params(scale=4, iterations=3, temporal_area_radius=1)
    want = _model(frames, _flows(3, 135, 240, seed=2), P)
    got, _ = _engine(frames, ListFlow(_flows(3, 135, 240, seed=2)), P)
    assert got[0].shape == (540 - 14, 960 - 14, 3)
    assert all(np.array_equal(g, wv) for g, wv in zip(got, want))


def test_graph_replay_params_and_streams():
    n, h, w = 5, 12, 16
    frames, flows = _frames(n, h, w, 3, seed=9), _flows(n, h, w, seed=9)
    P = M.Params(scale=2, iterations=5, temporal_area_radius=1)
    first, sr = _engine(frames, ListFlow(flows), P)
    # replay on the same handle (graphs captured by the first stream)
    sr.setOpticalFlow(ListFlow(flows))
    sr.setInput(frames)
    again = [sr.nextFrame(float_output=True).cpu().numpy() for _ in range(n)]
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
    eager, _ = _engine(frames, ListFlow(flows), P, use_graph=0)
    assert all(np.array_equal(a, b) for a, b in zip(first, eager))
    # changed then restored parameter equals a fresh handle
    sr.setIterations(7)
    sr.setLambda(0.1)
    sr.setOpticalFlow(ListFlow(flows))
    sr.setInput(frames)
    sr.nextFrame()
    sr.setIterations(5)
    sr.setLambda(0.03)
    sr.setOpticalFlow(ListFlow(flows))
    sr.setInput(frames)
    restored = [sr.nextFrame(float_output=True).cpu().numpy() for _ in range(n)]
    assert all(np.array_equal(a, b) for a, b in zip(first, restored))
    # two handles on two streams
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    frames2, flows2 = _frames(n, h, w, 3, seed=10), _flows(n, h, w, seed=10)
    serial2, _ = _engine(frames2, ListFlow(flows2), P)
    a, _ = _engine(frames, ListFlow(flows), P)
    ha, hb = ocb.createSuperResolution_BTVL1_CUDA(), ocb.createSuperResolution_BTVL1_CUDA()
    outs = {0: [], 1: []}
    for i, (hnd, fr, fl) in enumerate(((ha, frames, flows), (hb, frames2, flows2))):
        hnd.setOpticalFlow(ListFlow(fl))
        hnd.setScale(2), hnd.setIterations(5), hnd.setTemporalAreaRadius(1)
        hnd.setInput(fr)
    for _ in range(n):
        with torch.cuda.stream(s1):
            outs[0].append(ha.nextFrame(float_output=True, stream=s1))
        with torch.cuda.stream(s2):
            outs[1].append(hb.nextFrame(float_output=True, stream=s2))
    torch.cuda.synchronize()
    assert all(np.array_equal(x.cpu().numpy(), y) for x, y in zip(outs[0], a))
    assert all(np.array_equal(x.cpu().numpy(), y) for x, y in zip(outs[1], serial2))


def test_launches_per_output_frame():
    n, h, w, iters = 6, 10, 12, 20
    P = M.Params(scale=2, iterations=iters, temporal_area_radius=2)
    _, sr = _engine(_frames(n, h, w, 1, seed=4), ListFlow(_flows(n, h, w, seed=4)), P)
    K = 2 * P.temporal_area_radius + 1
    assert sr.getStats()["launches"] <= n * (2 * iters + 2 * K + 4)


def test_refused_arguments():
    l = _lib.lib()
    ok = lambda f: f == 0
    h = C.c_void_p()
    assert l.b2f_superres_create(None, None, None) == 1
    dis = ocb.DISOpticalFlow_create()
    assert l.b2f_superres_create(None, dis._h, C.byref(h)) == 1  # not a superres flow engine
    assert ok(l.b2f_superres_create(None, None, C.byref(h)))
    frame = torch.zeros((8, 8), dtype=torch.uint8, device=DEV)
    img = superres._image(frame)
    flt = torch.zeros((8, 8), dtype=torch.float32, device=DEV)
    fimg = superres._image(flt)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert l.b2f_superres_push(h, C.byref(img), s) == 1  # no flow engine: flows must be pushed
    for pid, bad in ((800, 1), (801, 0), (802, 0), (804, 0), (805, 0), (805, 17), (806, 0), (806, 4), (806, 33),
                     (807, -1), (808, -1), (808, 16)):
        d = C.c_double()
        l.b2f_superres_get_param(h, pid, C.byref(d))
        assert ok(l.b2f_superres_set_param(h, pid, bad))
        assert l.b2f_superres_push_flows(h, C.byref(img), None, None, None, None, s) == 1, pid
        assert ok(l.b2f_superres_set_param(h, pid, d.value))
    assert l.b2f_superres_set_param(h, 899, 1) == 1
    f16 = superres._image(torch.zeros((8, 8), dtype=torch.float32, device=DEV))
    assert l.b2f_superres_push_flows(h, C.byref(f16), None, None, None, None, s) == 2  # not 8UC1/3/4
    assert ok(l.b2f_superres_set_param(h, 800, 2))
    assert ok(l.b2f_superres_set_param(h, 808, 1))
    small = superres._image(torch.zeros((3, 3), dtype=torch.uint8, device=DEV))
    assert l.b2f_superres_push_flows(h, C.byref(small), None, None, None, None, s) == 1  # crop leaves no pixels
    got = C.c_int()
    assert l.b2f_superres_pop(h, None, C.byref(got), s) == 1  # no frame yet
    assert ok(l.b2f_superres_push_flows(h, C.byref(img), None, None, None, None, s))
    other = superres._image(torch.zeros((9, 8), dtype=torch.uint8, device=DEV))
    assert l.b2f_superres_push_flows(h, C.byref(other), C.byref(fimg), C.byref(fimg), C.byref(fimg), C.byref(fimg), s) == 3
    c3 = superres._image(torch.zeros((8, 8, 3), dtype=torch.uint8, device=DEV))
    assert l.b2f_superres_push_flows(h, C.byref(c3), C.byref(fimg), C.byref(fimg), C.byref(fimg), C.byref(fimg), s) == 2
    assert l.b2f_superres_push_flows(h, C.byref(img), None, None, None, None, s) == 1  # flows required after the first
    wrong = superres._image(torch.zeros((8, 9), dtype=torch.float32, device=DEV))
    assert l.b2f_superres_push_flows(h, C.byref(img), C.byref(wrong), C.byref(fimg), C.byref(fimg), C.byref(fimg), s) == 3
    assert ok(l.b2f_superres_push_flows(h, C.byref(img), C.byref(fimg), C.byref(fimg), C.byref(fimg), C.byref(fimg), s))
    assert ok(l.b2f_superres_push_flows(h, C.byref(img), C.byref(fimg), C.byref(fimg), C.byref(fimg), C.byref(fimg), s))
    w = C.c_int()
    assert ok(l.b2f_superres_wants_frame(h, C.byref(w))) and w.value == 1  # the first output reads 2R + 2 frames
    assert ok(l.b2f_superres_push_flows(h, C.byref(img), C.byref(fimg), C.byref(fimg), C.byref(fimg), C.byref(fimg), s))
    assert ok(l.b2f_superres_wants_frame(h, C.byref(w))) and w.value == 0
    assert l.b2f_superres_push_flows(h, C.byref(img), C.byref(fimg), C.byref(fimg), C.byref(fimg), C.byref(fimg), s) == 1
    out = superres._image(torch.zeros((3, 2), dtype=torch.uint8, device=DEV))
    assert l.b2f_superres_pop(h, C.byref(out), C.byref(got), s) == 3  # the output is 16 - 14 = 2 x 2
    out = superres._image(torch.zeros((2, 2), dtype=torch.int32, device=DEV).view(torch.float32))
    out.type = 13
    assert l.b2f_superres_pop(h, C.byref(out), C.byref(got), s) == 2  # wrong output type
    l.b2f_superres_destroy(h)
    # the wrappers
    fb = ocb.FarnebackOpticalFlow_create()
    a = superres._image(torch.zeros((8, 8, 3), dtype=torch.uint8, device=DEV))
    b = superres._image(torch.zeros((8, 8, 4), dtype=torch.uint8, device=DEV))
    fl = superres._image(torch.zeros((8, 8), dtype=torch.float32, device=DEV))
    assert l.b2f_calc_ext(fb._h, C.byref(a), C.byref(b), C.byref(fl), C.byref(fl), s) == 2
    assert l.b2f_calc_ext(dis._h, C.byref(a), C.byref(a), C.byref(fl), C.byref(fl), s) == 1
    assert l.b2f_calc_ext(fb._h, C.byref(a), C.byref(fimg), C.byref(fl), C.byref(fl), s) == 2


@pytest.mark.parametrize("R", [0, 1])
def test_mid_stream_parameter_changes(R):
    """btvKernelSize changed mid-stream takes effect at the next processed frame, as in the model (with R = 0 the output
    returned is the one processed in the same call); scale is read only when the stream starts."""
    n, h, w = 5, 10, 12
    frames, flows = _frames(n, h, w, 3, seed=20 + R), _flows(n, h, w, seed=20 + R)
    P = M.Params(scale=2, iterations=3, temporal_area_radius=R)
    it = iter(flows)
    m = M.BTVL1(M.ListSource(frames), lambda a, b: next(it), P)
    sr = ocb.createSuperResolution_BTVL1_CUDA()
    sr.setOpticalFlow(ListFlow(flows))
    sr.setScale(2), sr.setIterations(3), sr.setTemporalAreaRadius(R)
    sr.setInput(frames)
    for i in range(n):
        if i == 2:
            P.btv_kernel_size = 5
            sr.setKernelSize(5)
            sr.setScale(3)
        want = m.next_frame()
        got = sr.nextFrame(float_output=True).cpu().numpy()
        assert got.shape == want.shape and np.array_equal(got, want), i
    assert sr.nextFrame() is None and m.next_frame() is None
