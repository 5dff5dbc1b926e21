"""GPU tests of the VariationalRefinement engine (csrc/varref.cu): the refined flow bit for bit against the float32
model oracle/dis_model.py ``refine`` at the benchmark frame sizes, at the solver's region-tile edges for every
SOR-iterations-per-launch value its cost model picks, at one-pixel-thin shapes, across parameters, input types and
pitched buffers; and the engine contract: in-place refinement, planar and host forms, live parameter changes,
concurrent handles, the batch front end, status codes and the C++ adapter."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import synth, dis_model as D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_varref_compat")
SR = 64  # solver region edge (csrc/variational.cuh)
DEFAULTS = dict(fixed_point_iterations=5, sor_iterations=5, omega=1.6, alpha=20.0, delta=5.0, gamma=10.0,
                epsilon=0.001)
# the parameter sets tests/test_varref_model_cpu.py pins the model to cv2 with
PARAM_SETS = [
    DEFAULTS,
    dict(DEFAULTS, epsilon=0.01),
    dict(DEFAULTS, omega=1.0, sor_iterations=12),
    dict(DEFAULTS, fixed_point_iterations=2, sor_iterations=25, omega=1.9, epsilon=0.05),
    dict(DEFAULTS, fixed_point_iterations=1, sor_iterations=1, alpha=3.0, delta=0.5, gamma=1.0),
]
SETTERS = dict(fixed_point_iterations="FixedPointIterations", sor_iterations="SorIterations", omega="Omega",
               alpha="Alpha", delta="Delta", gamma="Gamma", epsilon="Epsilon")


def _alg(p=DEFAULTS):
    import opencv_contrib_b200 as ocb
    alg = ocb.VariationalRefinement_create()
    for k, v in p.items():
        getattr(alg, "set" + SETTERS[k])(v)
    return alg


def _case(h, w, seed, dtype="u8"):
    """A pair with smooth motion and an initial flow off the true one by up to 1 px."""
    I0, I1, gt = synth.make_pair(h, w, seed=seed, kind="smooth", mag=2.0, dtype=dtype)
    rng = np.random.default_rng(seed)
    flow = (gt + (rng.random(gt.shape) - 0.5) * 2).astype(np.float32)
    return I0, I1, flow


def _model(I0, I1, flow, p=DEFAULTS):
    u, v = D.refine(I0, I1, flow[..., 0], flow[..., 1], p["alpha"], p["delta"], p["gamma"], p["epsilon"], p["omega"],
                    p["fixed_point_iterations"], p["sor_iterations"], np.float32)
    return np.stack([u, v], -1)


def _run(dev, I0, I1, flow, alg=None, p=DEFAULTS):
    """One calc on a side stream (the CUDA-graph path); returns the refined flow and the handle."""
    import torch
    alg = alg or _alg(p)
    s = torch.cuda.Stream(device=dev)
    f = torch.from_numpy(flow).to(dev)
    with torch.cuda.stream(s):
        out = alg.calc(torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev), f, stream=s)
    s.synchronize()
    assert out is f  # refined in place
    return out.cpu().numpy(), alg


def _same(got, want):
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (
        int((got != want).any(axis=-1).sum()), float(np.nanmax(np.abs(got - want))))


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _iters_per_launch(h, w, n, sms):
    """The engine's launch-cost model (variational_iters_per_launch in csrc/variational.cuh)."""
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


def _edge_shapes(sms):
    """(h, w, sor, k) for every SOR-iterations-per-launch k the cost model picks at 5 and 25 SOR iterations (the
    benchmark's) on frames from 160x120 to 4K, each taken at the smallest frame that picks it: both sides at m * t - 1,
    m * t and m * t + 1 for the tile t = 64 - 4 k, m from that frame, searched to the nearest multiples at which the
    model still picks k."""
    picked = {}
    for sor in (5, 25):
        for h, w in ((120, 160), (240, 320), (480, 640), (1080, 1920), (2160, 3840)):
            picked.setdefault(_iters_per_launch(h, w, sor, sms), (h, w, sor))
    out = set()
    for k, (h, w, sor) in picked.items():
        t = SR - 4 * k
        mh, mw = max(1, round(h / t)), max(1, round(w / t))
        cands = [(mh + a, mw + b) for a in (0, -1, 1, -2, 2) for b in (0, -1, 1, -2, 2)]
        for d in (-1, 0, 1):
            for a, b in cands:
                hh, ww = a * t + d, b * t + d
                if hh > 0 and ww > 0 and _iters_per_launch(hh, ww, sor, sms) == k:
                    out.add((hh, ww, sor, k))
                    break
    return sorted(out)


def _check(dev, h, w, p=DEFAULTS, seed=None, k=None):
    I0, I1, flow = _case(h, w, h * 7 + w if seed is None else seed)
    got, alg = _run(dev, I0, I1, flow, p=p)
    assert np.isfinite(got).all()
    _same(got, _model(I0, I1, flow, p))
    st = alg.getStats()
    assert st["levels"] == 1 and st["iterations_run"] == p["fixed_point_iterations"] * p["sor_iterations"]
    assert alg.getActivePath() == _iters_per_launch(h, w, p["sor_iterations"], _sms())
    if k is not None:
        assert alg.getActivePath() == k


@pytest.mark.parametrize("h,w", [(480, 640), (1080, 1920)])
def test_benchmark_sizes_match_model_bit_for_bit(cuda_device, h, w):
    _check(cuda_device, h, w, seed=1)


def test_region_tile_edges_match_model_bit_for_bit(cuda_device):
    """Shapes one pixel either side of whole tiles for every k the cost model picks (sor 25 also leaves a shorter last
    launch), and the single-region boundary: 64x64 runs the single-CTA kernel, 65x64 and 64x65 the region solver."""
    shapes = _edge_shapes(_sms())
    assert len({k for _, _, _, k in shapes}) >= 2, shapes
    for h, w, sor, k in shapes:
        _check(cuda_device, h, w, dict(DEFAULTS, fixed_point_iterations=1, sor_iterations=sor), k=k)
    for h, w in ((64, 64), (65, 64), (64, 65)):
        _check(cuda_device, h, w)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 200), (200, 1), (2, 130), (1, 7), (7, 1)])
def test_thin_shapes_match_model_bit_for_bit(cuda_device, h, w):
    """cv2 accepts frames one pixel high or wide; DeepFlow and DIS never run levels this thin."""
    _check(cuda_device, h, w)
    _check(cuda_device, h, w, dict(DEFAULTS, sor_iterations=25))


def _pitched(dev, a, pad, dtype=None):
    """A view of `a` on the device inside a wider buffer: rows pitched, first column offset."""
    import torch
    t = torch.from_numpy(a).to(dev)
    shape = (a.shape[0], a.shape[1] + 2 * pad) + a.shape[2:]
    big = torch.full(shape, 7, dtype=t.dtype, device=dev)
    big[:, pad:pad + a.shape[1]] = t
    return big[:, pad:pad + a.shape[1]]


@pytest.mark.parametrize("p", PARAM_SETS, ids=range(len(PARAM_SETS)))
@pytest.mark.parametrize("dtype", ["u8", "f32"])
def test_parameters_types_and_pitched_buffers_match_model(cuda_device, p, dtype):
    import torch
    h, w = 70, 90
    I0, I1, flow = _case(h, w, 3, dtype)
    want = _model(I0, I1, flow, p)
    got, _ = _run(cuda_device, I0, I1, flow, p=p)
    _same(got, want)
    alg = _alg(p)
    f = _pitched(cuda_device, flow, 5)
    assert f.stride(0) > 2 * w
    out = alg.calc(_pitched(cuda_device, I0, 13), _pitched(cuda_device, I1, 3), f)  # NULL stream: no graph
    _same(out.cpu().numpy(), want)
    u, v = _pitched(cuda_device, flow[..., 0].copy(), 9), _pitched(cuda_device, flow[..., 1].copy(), 2)
    alg.calcUV(_pitched(cuda_device, I0, 13), _pitched(cuda_device, I1, 3), u, v)
    torch.cuda.synchronize()
    _same(np.stack([u.cpu().numpy(), v.cpu().numpy()], -1), want)


def test_u8_frames_and_their_float_copies_alike(cuda_device):
    I0, I1, flow = _case(96, 120, 12)
    got, _ = _run(cuda_device, I0, I1, flow)
    _same(_run(cuda_device, I0.astype(np.float32), I1.astype(np.float32), flow)[0], got)


def test_calc_uv_and_calc_host_equal_calc(cuda_device):
    import torch
    I0, I1, flow = _case(100, 150, 5)
    want, alg = _run(cuda_device, I0, I1, flow)
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    u = torch.from_numpy(flow[..., 0].copy()).to(cuda_device)
    v = torch.from_numpy(flow[..., 1].copy()).to(cuda_device)
    ru, rv = alg.calcUV(d0, d1, u, v)
    torch.cuda.synchronize()
    assert ru is u and rv is v
    _same(np.stack([u.cpu().numpy(), v.cpu().numpy()], -1), want)
    host = flow.copy()
    assert alg.calc_host(I0, I1, host) is host
    _same(host, want)


def test_no_step_returns_the_flow(cuda_device):
    """An iteration count below one (or omega 0) runs no step, as in cv2: the flow comes back with its values."""
    I0, I1, flow = _case(80, 100, 6)
    for change in (dict(fixed_point_iterations=0), dict(fixed_point_iterations=-3), dict(sor_iterations=0),
                   dict(sor_iterations=-1), dict(omega=0.0)):
        p = dict(DEFAULTS, **change)
        got, alg = _run(cuda_device, I0, I1, flow, p=p)
        assert np.array_equal(got, flow), change
        _same(got, _model(I0, I1, flow, p))
        assert alg.getStats()["iterations_run"] == max(0, p["fixed_point_iterations"]) * max(0, p["sor_iterations"])


def test_parameter_change_on_a_live_handle_matches_a_fresh_one(cuda_device):
    I0, I1, flow = _case(90, 130, 7)
    alg = _alg()
    _run(cuda_device, I0, I1, flow, alg=alg)  # captures the defaults' graph
    p = PARAM_SETS[3]
    for k, v in p.items():
        getattr(alg, "set" + SETTERS[k])(v)
        assert getattr(alg, "get" + SETTERS[k])() == pytest.approx(v)
    got, _ = _run(cuda_device, I0, I1, flow, alg=alg)
    _same(got, _run(cuda_device, I0, I1, flow, p=p)[0])
    _same(got, _model(I0, I1, flow, p))


def test_handles_on_concurrent_streams_equal_a_sequential_run(cuda_device):
    import torch
    n = 4
    cases = [_case(120, 160, 20 + i) for i in range(n)]
    want = [_run(cuda_device, *c)[0] for c in cases]
    algs = [_alg() for _ in range(n)]
    streams = [torch.cuda.Stream(device=cuda_device) for _ in range(n)]
    ins = [(torch.from_numpy(a).to(cuda_device), torch.from_numpy(b).to(cuda_device)) for a, b, _ in cases]
    torch.cuda.synchronize()
    for _ in range(2):  # capture, then replay
        flows = [torch.from_numpy(c[2]).to(cuda_device) for c in cases]
        torch.cuda.synchronize()
        for alg, s, (a, b), f in zip(algs, streams, ins, flows):
            alg.calc(a, b, f, stream=s)
        for s in streams:
            s.synchronize()
        for f, w in zip(flows, want):
            _same(f.cpu().numpy(), w)


def test_native_batch_algo_8_equals_pairwise(cuda_device):
    import torch
    from opencv_contrib_b200.batch import NativeFlowBatch
    cases = [_case(72, 96, 30 + i) for i in range(5)]
    p = dict(DEFAULTS, sor_iterations=6)
    want = [_run(cuda_device, *c, p=p)[0] for c in cases]
    nb = NativeFlowBatch("varref", dict(sor_iterations=6), n_streams=2)
    out = [c[2].copy() for c in cases]
    nb.run_host([(a, b) for a, b, _ in cases], out)
    flows = [torch.from_numpy(c[2]).to(cuda_device) for c in cases]
    nb.run_device([(torch.from_numpy(a).to(cuda_device), torch.from_numpy(b).to(cuda_device)) for a, b, _ in cases],
                  flows)
    torch.cuda.synchronize()
    nb.close()
    for i in range(5):
        _same(out[i], want[i])
        _same(flows[i].cpu().numpy(), want[i])


@pytest.mark.parametrize("h,w", [(40, 56), (96, 128)])
def test_a_nan_in_the_flow_gives_the_models_pattern(cuda_device, h, w):
    I0, I1, flow = _case(h, w, 8)
    flow[h // 2, w // 3, 0] = np.nan
    got, _ = _run(cuda_device, I0, I1, flow)
    with np.errstate(invalid="ignore"):
        want = _model(I0, I1, flow)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    assert np.array_equal(got[fin].view(np.uint32), want[fin].view(np.uint32))


def test_status_codes_video_refusal_and_name(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200 import _lib
    from opencv_contrib_b200.video import VideoFlow
    alg = _alg()
    assert alg.getDefaultName() == "my_object" and alg._needs_initial_flow()
    I0, I1, flow = _case(40, 50, 9)
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    f = torch.from_numpy(flow).to(cuda_device)
    with pytest.raises(ocb.B2FError) as e:  # the flow is always read: it must be given
        alg.calc(d0, d1)
    assert e.value.status == 1
    lib = _lib.lib()

    def status(a, b, fl):
        return lib.b2f_calc(alg._h, C.byref(a), C.byref(b), C.byref(fl), None)

    img = lambda t, typ, step: _lib.b2f_image(t.data_ptr(), step, t.shape[0], t.shape[1], typ)
    i0, i1 = img(d0, _lib.B2F_8UC1, 50), img(d1, _lib.B2F_8UC1, 50)
    fl = img(f, _lib.B2F_32FC2, 400)
    f32 = d1.float()
    assert status(i0, img(f32, _lib.B2F_32FC1, 200), fl) == 2  # mixed types
    assert status(img(d0, 2, 100), img(d1, 2, 100), fl) == 2  # 16UC1
    assert status(i0, i1, img(f, _lib.B2F_32FC1, 400)) == 2  # a flow that is not 32FC2
    small = _lib.b2f_image(d1.data_ptr(), 50, 39, 50, _lib.B2F_8UC1)
    assert status(i0, small, fl) == 3
    assert status(i0, i1, _lib.b2f_image(f.data_ptr(), 400, 40, 49, _lib.B2F_32FC2)) == 3
    assert status(i0, i1, fl) == 0
    torch.cuda.synchronize()
    _same(f.cpu().numpy(), _model(I0, I1, flow))
    with pytest.raises(ocb.B2FError) as e:
        VideoFlow(alg, 40, 50, dtype=np.uint8, depth=2, warm_start=False)
    assert e.value.status == 1
    with pytest.raises(ocb.B2FError):
        VideoFlow(alg, 40, 50, dtype=np.uint8, depth=2, warm_start=True)


def test_cpp_call_site_matches_model(cuda_device, tmp_path):
    rows, cols = 75, 130
    I0, I1, flow = _case(rows, cols, 10)
    paths = [tmp_path / n for n in ("i0.raw", "i1.raw", "flow.raw", "out.raw", "uv.raw")]
    I0.tofile(paths[0])
    I1.tofile(paths[1])
    flow.tofile(paths[2])
    r = subprocess.run([EXE, str(rows), str(cols)] + [str(p) for p in paths], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    want = _model(I0, I1, flow, dict(DEFAULTS, sor_iterations=7, epsilon=0.01))
    _same(np.fromfile(paths[3], np.float32).reshape(rows, cols, 2), want)
    uv = np.fromfile(paths[4], np.float32).reshape(2, rows, cols)
    _same(np.stack([uv[0], uv[1]], -1), want)
