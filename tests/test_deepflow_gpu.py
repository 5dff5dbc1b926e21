"""GPU tests of the DeepFlow engine (csrc/deepflow.cu): bit for bit against oracle/deepflow_model.py at shapes that hit
the solver's region and halo edges, the full pair against the live cv2 restatement (oracle/deepflow_ref.py) within
cv2's own last-bit sensitivity, accuracy on synthetic motion, and the engine contract."""
import math
import threading

import numpy as np
import pytest

from oracle import synth, metrics, deepflow_ref as R, deepflow_model as M

pytestmark = pytest.mark.gpu

SR = 64  # solver region edge (csrc/deepflow.cu)


def _alg(**kw):
    import opencv_contrib_b200 as ocb
    return ocb.createOptFlow_DeepFlow(**kw)


def _run(dev, I0, I1, alg=None, **kw):
    import torch
    alg = alg or _alg(**kw)
    f = alg.calc(torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev))
    torch.cuda.synchronize()
    return f.cpu().numpy(), alg


def _params(**kw):
    p = dict(sigma=0.6, min_size=25, downscale_factor=0.95, fixed_point_iterations=5, sor_iterations=25, alpha=1.0,
             delta=0.5, gamma=5.0, omega=1.6, max_layers=200)
    p.update(kw)
    return p


def _create_kw(p):
    return dict(sigma=p["sigma"], minSize=p["min_size"], downscaleFactor=p["downscale_factor"],
                fixedPointIterations=p["fixed_point_iterations"], sorIterations=p["sor_iterations"], alpha=p["alpha"],
                delta=p["delta"], gamma=p["gamma"], omega=p["omega"], maxLayers=p["max_layers"])


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _iters_per_launch(h, w, n, sms):
    """The engine's launch-cost model (DeepFlowEngine::iters_per_launch)."""
    if w <= SR and h <= SR:
        return n
    best, best_it = 1e30, 1
    for cand in range(1, min(12, n) + 1):
        t = SR - 4 * cand
        if t < 8:
            break
        cost = math.ceil(n / cand) * (math.ceil(math.ceil(w / t) * math.ceil(h / t) / sms) * (3.0 + 0.7 * cand) + 2.0)
        if cost < best:
            best, best_it = cost, cand
    return best_it


def _edge_shapes(sor, sms):
    """Single-level (h, w, k) shapes for every k the cost model picks, at this SM count and `sor`, on the levels of the
    640x480 and 1080p pyramids: each side at m * t - 1, m * t and m * t + 1 for the tile t = 64 - 4 k, with m taken from
    the level the k was picked on (so multi-wave shapes keep their k), searched to the nearest multiples at which the
    model still picks k.  Plus the one-region boundary and the smallest levels."""
    picked = {}
    for H, W in ((480, 640), (1080, 1920)):
        for h, w in R.pyramid_sizes(H, W):
            if h > SR or w > SR:
                picked.setdefault(_iters_per_launch(h, w, sor, sms), (h, w))
    out = set()
    for k, (h, w) in picked.items():
        t = SR - 4 * k
        mh, mw = max(1, round(h / t)), max(1, round(w / t))
        cands = [(mh + a, mw + b) for a in (0, -1, 1, -2, 2) for b in (0, -1, 1, -2, 2)]
        for d in (-1, 0, 1):
            for a, b in cands:
                hh, ww = a * t + d, b * t + d
                if hh > 0 and ww > 0 and _iters_per_launch(hh, ww, sor, sms) == k:
                    out.add((hh, ww, k))
                    break
    for h, w in ((26, 30), (64, 64), (65, 64), (64, 65), (1, 40), (40, 2)):
        out.add((h, w, _iters_per_launch(h, w, sor, sms)))
    return sorted(out)


def _check_single_level(dev, h, w, fp, sor, k=None, seed=None):
    I0, I1, _ = synth.make_pair(h, w, seed=h * 7 + w if seed is None else seed, kind="smooth", mag=2.0)
    p = _params(max_layers=0, fixed_point_iterations=fp, sor_iterations=sor)
    want = M.calc(I0, I1, R.DeepFlowParams(**p))
    got, alg = _run(dev, I0, I1, **_create_kw(p))
    assert alg.getStats()["levels"] == 1
    assert np.isfinite(got).all()
    assert np.array_equal(got, want), (int((got != want).any(axis=-1).sum()), float(np.abs(got - want).max()))
    assert alg.getActivePath(0) == _iters_per_launch(h, w, sor, _sms())
    if k is not None:
        assert alg.getActivePath(0) == k


@pytest.mark.parametrize("fp,sor", [(1, 1), (2, 25), (1, 10)])
def test_single_level_region_edges_match_model_bit_for_bit(cuda_device, fp, sor):
    """One level (max_layers 0): warp + derivatives, system terms and the solver, at shapes one pixel either side of
    whole tiles for every iterations-per-launch k the benchmark pyramids use (k iterations per launch must equal the
    model's one sweep at a time; sor 25 also leaves a shorter last launch)."""
    shapes = _edge_shapes(sor, _sms())
    if sor > 1:
        assert len({k for _, _, k in shapes}) >= 2, shapes
    for h, w, k in shapes:
        _check_single_level(cuda_device, h, w, fp, sor, k)


@pytest.mark.parametrize("h,w", [(480, 640), (1080, 1920)])
def test_single_level_benchmark_size_matches_model_bit_for_bit(cuda_device, h, w):
    _check_single_level(cuda_device, h, w, 2, 25, seed=1)


@pytest.mark.parametrize("h,w,dtype", [(96, 128, "u8"), (75, 131, "f32"), (140, 67, "u8")])
def test_pyramid_matches_model_bit_for_bit(cuda_device, h, w, dtype):
    I0, I1, _ = synth.make_pair(h, w, seed=11, kind="affine", dtype=dtype)
    p = _params(sor_iterations=10)
    want = M.calc(I0, I1, R.DeepFlowParams(**p))
    got, alg = _run(cuda_device, I0, I1, **_create_kw(p))
    assert np.array_equal(got, want), (int((got != want).any(axis=-1).sum()), float(np.abs(got - want).max()))
    sizes = R.pyramid_sizes(h, w, R.DeepFlowParams(**p))
    assert alg.getStats()["levels"] == len(sizes)
    for l, (r, c) in enumerate(sizes):
        assert alg.getActivePath(l) == _iters_per_launch(r, c, 10, _sms())


def _yardstick(I0, I1):
    base = R.calc(I0, I1)
    pert = (I1.astype(np.float32) * np.float32(1 + 1e-6)).astype(np.float32)
    e = metrics.epe(R.calc(I0, pert), base)
    return base, float(e.mean()), float(np.quantile(e, 0.99))


@pytest.mark.parametrize("h,w", [(480, 640), (1080, 1920)])
def test_full_pair_within_cv2_sensitivity(cuda_device, h, w):
    I0, I1, _ = synth.make_pair(h, w, seed=1, kind="smooth", mag=4.0)
    base, mean_y, p99_y = _yardstick(I0, I1)
    got, alg = _run(cuda_device, I0, I1)
    assert alg.getStats()["levels"] == len(R.pyramid_sizes(h, w))
    e = metrics.epe(got, base)
    assert e.mean() <= 4 * mean_y and np.quantile(e, 0.99) <= 4 * p99_y, (float(e.mean()), mean_y,
                                                                           float(np.quantile(e, 0.99)), p99_y)


def test_accuracy_constant_shift(cuda_device):
    I0, I1, gt = synth.make_pair(480, 640, seed=0, kind="const")
    got, _ = _run(cuda_device, I0, I1)
    e = metrics.epe(got, gt)
    assert e.mean() <= 0.06, float(e.mean())
    assert (e[16:-16, 16:-16] <= 0.1).mean() >= 0.999


@pytest.mark.parametrize("kind", ["affine", "smooth"])
def test_accuracy_like_cv2(cuda_device, kind):
    I0, I1, gt = synth.make_pair(480, 640, seed=2, kind=kind, mag=4.0)
    ref = metrics.epe(R.calc(I0, I1), gt)
    e = metrics.epe(_run(cuda_device, I0, I1)[0], gt)
    assert e.mean() <= 1.1 * ref.mean() + 1e-3, (float(e.mean()), float(ref.mean()))
    assert np.quantile(e, 0.99) <= 1.1 * np.quantile(ref, 0.99) + 1e-3


def test_repeat_graph_threads_bit_identical(cuda_device):
    import torch
    I0, I1, _ = synth.make_pair(120, 160, seed=4, kind="smooth")
    p = _create_kw(_params(sor_iterations=8))
    eager, _ = _run(cuda_device, I0, I1, alg=_set_graph(_alg(**p), 0))
    alg = _alg(**p)
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    s = torch.cuda.Stream(device=cuda_device)
    outs = []
    with torch.cuda.stream(s):
        for _ in range(3):  # capture, then replays
            outs.append(alg.calc(d0, d1, stream=s))
    s.synchronize()
    for o in outs:
        assert np.array_equal(o.cpu().numpy(), eager)
    res = [None] * 4

    def work(k):
        torch.cuda.set_device(cuda_device)
        st = torch.cuda.Stream(device=cuda_device)
        a = _alg(**p)
        with torch.cuda.stream(st):
            f = a.calc(d0, d1, stream=st)
            f2 = a.calc(d0, d1, stream=st)
        st.synchronize()
        res[k] = (f.cpu().numpy(), f2.cpu().numpy())

    ts = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in res:
        assert np.array_equal(r[0], eager) and np.array_equal(r[1], eager)


def _set_graph(alg, on):
    alg.setEngineOption("use_graph", on)
    return alg


def test_pitched_inputs_null_stream_and_errors(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(70, 90, seed=6, kind="smooth")
    want, alg = _run(cuda_device, I0, I1, sorIterations=5)
    b0 = torch.zeros((70, 160), dtype=torch.uint8, device=cuda_device)
    b1 = torch.zeros((70, 128), dtype=torch.uint8, device=cuda_device)
    b0[:, 13:103] = torch.from_numpy(I0).to(cuda_device)
    b1[:, 5:95] = torch.from_numpy(I1).to(cuda_device)
    flow = alg.calc(b0[:, 13:103], b1[:, 5:95])  # NULL stream: synchronised on return
    assert np.array_equal(flow.cpu().numpy(), want)
    u, v = alg.calcUV(b0[:, 13:103], b1[:, 5:95])
    torch.cuda.synchronize()
    assert np.array_equal(u.cpu().numpy(), want[..., 0]) and np.array_equal(v.cpu().numpy(), want[..., 1])
    assert np.array_equal(alg.calc_host(I0, I1), want)
    d0 = torch.from_numpy(I0).to(cuda_device)
    with pytest.raises(ocb.B2FError):  # mixed types
        alg.calc(d0, torch.from_numpy(I1.astype(np.float32)).to(cuda_device))
    with pytest.raises(ocb.B2FError):  # size mismatch
        alg.calc(d0, torch.from_numpy(I1[:, :80].copy()).to(cuda_device))
    with pytest.raises(ocb.B2FError):  # unsupported type
        alg.calc(d0.to(torch.int32), torch.from_numpy(I1).to(cuda_device).to(torch.int32))
    assert alg.getDefaultName() == "DenseOpticalFlow.DeepFlow"
    assert alg.workspaceBytes(70, 90) > 0


def test_video_refuses_warm_start_and_runs_without(cuda_device):
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200.video import VideoFlow
    alg = _alg(sorIterations=5)
    with pytest.raises(ocb.B2FError):
        VideoFlow(alg, 64, 80, dtype=np.uint8, depth=2, warm_start=True)
    frames = [synth.make_pair(64, 80, seed=s, kind="smooth")[0] for s in range(4)]
    vf = VideoFlow(alg, 64, 80, dtype=np.uint8, depth=2, warm_start=False)
    flows = dict(vf.run(frames))
    vf.close()
    ref = _alg(sorIterations=5)
    assert sorted(flows) == [0, 1, 2]
    for k in range(3):
        assert np.array_equal(flows[k], ref.calc_host(frames[k], frames[k + 1])), k


def test_native_batch_algo_5_equals_pairwise(cuda_device):
    from opencv_contrib_b200.batch import NativeFlowBatch
    frames = [synth.make_pair(72, 96, seed=s, kind="smooth")[0] for s in range(5)]
    pairs = [(frames[i], frames[i + 1]) for i in range(4)]
    ref = _alg(sorIterations=6)
    want = [ref.calc_host(a, b) for a, b in pairs]
    nb = NativeFlowBatch("deepflow", dict(sor_iterations=6), n_streams=2)
    out = [np.zeros((72, 96, 2), np.float32) for _ in range(4)]
    nb.run_host(pairs, out)
    nb.close()
    for i in range(4):
        assert np.array_equal(out[i], want[i]), i


def test_stats_count_solver_launches(cuda_device):
    I0, I1, _ = synth.make_pair(96, 128, seed=8, kind="smooth")
    got, alg = _run(cuda_device, I0, I1)
    sor = alg.getStats()["classes"]["deepflow_sor"]
    assert sor["launches"] > 0 and sor["bytes"] > 0
