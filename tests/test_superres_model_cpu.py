"""CPU checks of the BTV-L1 super-resolution model (oracle/superres_model.c / .py): its primitives against live cv2, its
pull schedule against an independent transcription of btv_l1_cuda.cpp's loops, and its quality on a degraded synthetic
sequence by the reference's accuracy recipe (modules/superres/test/test_superres.cpp:137-273)."""
import cv2
import numpy as np
import pytest

from oracle import superres_model as M


def test_gray_rule_equals_cvtcolor_on_every_bgr_value():
    v = np.arange(1 << 24, dtype=np.uint32)
    bgr = np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(M.gray(bgr, False), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))
    bgra = np.concatenate([bgr, np.full(bgr.shape[:2] + (1,), 77, np.uint8)], -1)
    assert np.array_equal(M.gray(bgra, False), cv2.cvtColor(bgra, cv2.COLOR_BGRA2GRAY))
    # Brox's work type: x float(1/255), not x / 255
    g = M.gray(bgr[:1, :256], True)
    want = (np.float32(1.0 / 255.0) * cv2.cvtColor(bgr[:1, :256], cv2.COLOR_BGR2GRAY).astype(np.float32))
    assert np.array_equal(g, want)


@pytest.mark.parametrize("sigma", [0.0, 1.3])
def test_gaussian_taps_equal_cv2(sigma):
    for n in range(1, 32, 2):
        assert np.array_equal(M.gaussian_kernel(n, sigma), cv2.getGaussianKernel(n, sigma, cv2.CV_32F).ravel()), n


@pytest.mark.parametrize("n,sigma,cn", [(5, 0.0, 1), (7, 1.3, 3), (31, 0.0, 4), (3, 0.0, 1)])
def test_separable_blur_matches_sepfilter2d(n, sigma, cn):
    rng = np.random.default_rng(n)
    a = rng.uniform(-2, 2, (37, 53, cn)).astype(np.float32)
    got = M.sep_filter(a, n, sigma)
    k = cv2.getGaussianKernel(n, sigma, cv2.CV_32F)
    want = cv2.sepFilter2D(a, cv2.CV_32F, k, k, borderType=cv2.BORDER_REFLECT_101).reshape(a.shape)
    assert np.abs(got - want).max() <= 4 * np.spacing(np.float32(2))


def _schedule(N, R):
    """btv_l1_cuda.cpp:483-582 as plain index arithmetic: (idx, start, end, base) per processFrame, and per output the
    frame whose result the output ring's slot holds when it is returned (2R + 1 slots; with R = 0 the processFrame of the
    same call has already overwritten it)."""
    L = 2 * R + 1
    store = min(L, N) - 1
    log = [(i, 0, min(2 * R, store), i) for i in range(R + 1) if i <= store]
    slot = {i % L: i for i, _, _, _ in log}
    proc, out, outs = R, -1, []
    while out < store:
        store = min(store + 1, N - 1)
        if proc < store:
            proc += 1
            s = max(proc - R, 0)
            log.append((proc, s, min(s + 2 * R, store), proc - s))
            slot[proc % L] = proc
        out += 1
        outs.append(slot[out % L])
    return log, outs


@pytest.mark.parametrize("R", [0, 1, 2, 4])
def test_schedule_matches_transcription(R, monkeypatch):
    calls = []
    # each processed result is filled with its base frame's index, so an output names the frame it came from
    monkeypatch.setattr(M, "process", lambda src, fwd, bwd, base, P: calls.append(len(src)) or
                        np.full((2 * P.btv_kernel_size + 1,) * 2 + (1,), src[base][0, 0], np.float32))
    for N in sorted({R + 1, 2 * R + 1, 2 * R + 2, 3 * R + 5}):
        frames = [np.full((2, 2), i, np.uint8) for i in range(N)]
        P = M.Params(temporal_area_radius=R)
        outs, log = M.run(frames, lambda a, b: (np.zeros((2, 2), np.float32),) * 2, P)
        want_log, want_outs = _schedule(N, R)
        assert log == want_log, (N, R)
        assert len(outs) == len(want_outs) == N
        assert [int(o[0, 0]) for o in outs] == want_outs, (N, R)
        assert calls[-len(log):] == [e - s + 1 for _, s, e, _ in log]


def _mssim(a, b):
    """The reference's MSSIM (test_superres.cpp:69-133), averaged over all channels."""
    C1, C2 = 6.5025, 58.5225
    a, b = a.astype(np.float64), b.astype(np.float64)
    g = lambda x: cv2.GaussianBlur(x, (11, 11), 1.5)
    mu1, mu2 = g(a), g(b)
    s1, s2, s12 = g(a * a) - mu1 ** 2, g(b * b) - mu2 ** 2, g(a * b) - mu1 * mu2
    ssim = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 ** 2 + mu2 ** 2 + C1) * (s1 + s2 + C2))
    return float(ssim.mean())


def test_quality_on_degraded_sequence():
    """Textured sequence moving (-0.7, -0.45) high-resolution pixels per frame, degraded as DegradeFrameSource does
    (GaussianBlur 5x5, INTER_NEAREST down 2, Gaussian noise sigma 10, spikes 1/500), restored with ground-truth flows at
    scale 2, 100 iterations, R = 2.  Measured when written: 0.897 against 0.802 for cv2's cubic upscale of each degraded
    frame; the bar is the reference's 0.5 and a 0.05 lead over the cubic upscale."""
    rng = np.random.default_rng(7)
    H, W, N, s = 96, 96, 6, 2
    base = cv2.resize(rng.uniform(0, 255, (H // 4 + 8, W // 4 + 8)).astype(np.float32), (W + 32, H + 32),
                      interpolation=cv2.INTER_CUBIC)
    base = cv2.GaussianBlur(base, (0, 0), 1.0)
    d = np.array([0.7, 0.45])
    gold, lr = [], []
    for t in range(N):
        M_ = np.float32([[1, 0, 16 - d[0] * t], [0, 1, 16 - d[1] * t]])
        g = np.clip(cv2.warpAffine(base, M_, (W, H), flags=cv2.INTER_CUBIC), 0, 255).astype(np.uint8)
        gold.append(g)
        b = cv2.GaussianBlur(g, (5, 5), 0)
        small = cv2.resize(b, (W // s, H // s), interpolation=cv2.INTER_NEAREST).astype(np.float32)
        small += rng.normal(0, 10, small.shape)
        spikes = rng.random(small.shape) < 1 / 500
        small[spikes] = rng.integers(0, 256, spikes.sum())
        lr.append(np.clip(small, 0, 255).astype(np.uint8))
    calls = iter(range(2 * N))

    def flow(a, b):
        sign = -1 if next(calls) % 2 == 0 else 1  # reads alternate calc(prev, cur), calc(cur, prev)
        return (np.full(a.shape, sign * d[0] / s, np.float32), np.full(a.shape, sign * d[1] / s, np.float32))

    P = M.Params(scale=s, iterations=100, temporal_area_radius=2)
    outs, _ = M.run(lr, flow, P)
    k = P.btv_kernel_size
    crop = lambda a: a[k:a.shape[0] - k, k:a.shape[1] - k]
    got = np.mean([_mssim(M.to_u8(o), crop(g)) for o, g in zip(outs, gold)])
    cubic = np.mean([_mssim(crop(cv2.resize(f, (W, H), interpolation=cv2.INTER_CUBIC)), crop(g)) for f, g in zip(lr, gold)])
    assert got >= 0.5 and got >= cubic + 0.05, (got, cubic)
