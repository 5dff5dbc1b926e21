"""GPU tests of the DIS engine (csrc/dis.cu): bit for bit against oracle/dis_model.py on whole presets, at patch-grid
edges, with every option, on levels that take each refinement solver path and on pitched views; statistically against
the live cv2.DISOpticalFlow (whose CPU propagation differs from the engine's OpenCL one); and the engine contract."""
import threading

import numpy as np
import pytest

from oracle import synth, dis_model as M

pytestmark = pytest.mark.gpu

SR = 64  # the refinement solver's region edge (csrc/variational.cuh)


def _alg(p: M.DISParams):
    import opencv_contrib_b200 as ocb
    a = ocb.DISOpticalFlow_create(ocb.DISOPTICAL_FLOW_PRESET_FAST)
    a.setFinestScale(p.finest_scale)
    a.setCoarsestScale(p.coarsest_scale)
    a.setPatchSize(p.patch_size)
    a.setPatchStride(p.patch_stride)
    a.setGradientDescentIterations(p.grad_descent_iterations)
    a.setVariationalRefinementIterations(p.variational_refinement_iterations)
    a.setVariationalRefinementAlpha(p.alpha)
    a.setVariationalRefinementDelta(p.delta)
    a.setVariationalRefinementGamma(p.gamma)
    a.setVariationalRefinementEpsilon(p.epsilon)
    a.setUseMeanNormalization(p.use_mean_normalization)
    a.setUseSpatialPropagation(p.use_spatial_propagation)
    return a


def _run(dev, I0, I1, p, alg=None, stream=None, flow=None):
    import torch
    alg = alg or _alg(p)
    fl = None if flow is None else torch.from_numpy(flow.copy()).to(dev)
    f = alg.calc(torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev), fl, stream=stream)
    torch.cuda.synchronize()
    return f.cpu().numpy(), alg


def _assert_bits(got, want):
    assert got.shape == want.shape
    d = np.abs(got - want)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
        f"{int((got != want).sum())} of {got.size} differ, max {d.max()}"


@pytest.mark.parametrize("preset", [0, 1, 2])
@pytest.mark.parametrize("shape", [(480, 640), (1080, 1920)])
def test_presets_bit_exact(cuda_device, preset, shape):
    I0, I1, _ = synth.make_pair(*shape, seed=preset, kind="smooth", mag=5.0)
    import opencv_contrib_b200 as ocb
    alg = ocb.DISOpticalFlow_create(preset)
    got, alg = _run(cuda_device, I0, I1, None, alg)
    _assert_bits(got, M.calc(I0, I1, M.preset(preset)))


def _edge_shapes(stride):
    """Single-level sides with (n - 8) % stride = 0, 1 and stride - 1, and one with a single patch (n = 8..8 + stride - 1)."""
    out = []
    for r in (0, 1, stride - 1):
        out.append(8 + 20 * stride + r)
    out.append(8 + stride - 1)
    return out


@pytest.mark.parametrize("stride", [3, 4])
def test_patch_grid_edges(cuda_device, stride):
    sides = _edge_shapes(stride)
    for k, (h, w) in enumerate([(sides[0], sides[1]), (sides[2], sides[0]), (sides[3], sides[1]), (sides[1], sides[3])]):
        I0, I1, _ = synth.make_pair(h, w, seed=10 + k, kind="smooth", mag=2.0)
        p = M.DISParams(finest_scale=0, coarsest_scale=0, patch_stride=stride)
        got, alg = _run(cuda_device, I0, I1, p)
        _assert_bits(got, M.calc(I0, I1, p))
        hs, ws = M.grid(h, w, 8, stride)
        assert alg.getActivePath(0)[:2] == (ws, hs)


def test_finest_scale_5_area_table(cuda_device):
    """At finest scale 5 a 287x800 frame needs 37 row weights in the first area resize (ratio 287 / 8)."""
    I0, I1, _ = synth.make_pair(287, 800, seed=12, kind="smooth", mag=6.0)
    p = M.DISParams(finest_scale=5, variational_refinement_iterations=2)
    assert max(len(t) for t in M._area_tab(287, 287 >> 5)) > 34
    got, _ = _run(cuda_device, I0, I1, p)
    _assert_bits(got, M.calc(I0, I1, p))


@pytest.mark.parametrize("p", [M.DISParams(finest_scale=0, coarsest_scale=0, use_spatial_propagation=False),
                               M.DISParams(finest_scale=0, coarsest_scale=0), M.preset(1), M.preset(2)],
                         ids=["one-level", "one-level-prop", "fast", "medium"])
def test_initial_flow_bit_exact(cuda_device, p):
    I0, I1, gt = synth.make_pair(240, 320, seed=13, kind="smooth", mag=3.0)
    F = (gt * np.float32(1.1)).astype(np.float32)
    alg = _alg(p)
    alg.setUseInitialFlow(True)
    got, _ = _run(cuda_device, I0, I1, p, alg, flow=F)
    _assert_bits(got, M.calc(I0, I1, p, flow=F))
    assert not np.array_equal(got, M.calc(I0, I1, p))


def test_video_warm_start_chains_the_previous_flow(cuda_device):
    import opencv_contrib_b200 as ocb
    frames = [synth.make_pair(120, 168, seed=30 + k, kind="const")[0] for k in range(5)]
    p = M.preset(1)
    want, flow = [], None
    for k in range(4):
        flow = M.calc(frames[k], frames[k + 1], p, flow=flow) if k else M.calc(frames[k], frames[k + 1], p)
        want.append(flow)
    alg = ocb.DISOpticalFlow_create(1)
    vf = ocb.VideoFlow(alg, 120, 168, dtype=np.uint8, depth=2, warm_start=True)
    got = dict(vf.run(frames))
    vf.close()
    for k in range(4):
        _assert_bits(got[k], want[k])
    assert not alg.getUseInitialFlow()  # the front end restores the setting


@pytest.mark.parametrize("prop", [True, False])
@pytest.mark.parametrize("mean_norm", [True, False])
@pytest.mark.parametrize("gd", [1, 16])
def test_options_bit_exact(cuda_device, prop, mean_norm, gd):
    I0, I1, _ = synth.make_pair(240, 320, seed=4, kind="affine")
    p = M.DISParams(finest_scale=1, use_spatial_propagation=prop, use_mean_normalization=mean_norm,
                    grad_descent_iterations=gd, variational_refinement_iterations=2)
    got, _ = _run(cuda_device, I0, I1, p)
    _assert_bits(got, M.calc(I0, I1, p))


@pytest.mark.parametrize("shape", [(60, 64), (200, 260)])
def test_refinement_paths(cuda_device, shape):
    """A level that fits one solver region (one-launch path) and one that takes the multi-region solver."""
    I0, I1, _ = synth.make_pair(*shape, seed=5, kind="smooth", mag=2.0)
    p = M.DISParams(finest_scale=0, coarsest_scale=0, variational_refinement_iterations=5)
    got, alg = _run(cuda_device, I0, I1, p)
    _assert_bits(got, M.calc(I0, I1, p))
    it = alg.getActivePath(0)[2]
    if shape[0] <= SR and shape[1] <= SR:
        assert it == M.REFINE_SOR_ITERATIONS
    else:
        assert 1 <= it <= M.REFINE_SOR_ITERATIONS


def test_active_path_per_level(cuda_device):
    I0, I1, _ = synth.make_pair(480, 640, seed=6)
    import opencv_contrib_b200 as ocb
    _, alg = _run(cuda_device, I0, I1, None, ocb.DISOpticalFlow_create(1))
    sizes = M.level_sizes(480, 640, M.preset(1))
    for k, (h, w) in enumerate(sizes):
        ws, hs, it = alg.getActivePath(2 + k)
        assert (hs, ws) == M.grid(h, w, 8, 4)
        assert it >= 1
    with pytest.raises(Exception):
        alg.getActivePath(0)  # scale 0 is below the finest
    assert alg.getStats()["levels"] == len(sizes)
    assert alg.getDefaultName() == "my_object"


def test_pitched_views(cuda_device):
    import torch
    I0, I1, _ = synth.make_pair(150, 200, seed=7, kind="smooth", mag=3.0)
    p = M.DISParams(finest_scale=1)
    B0 = torch.zeros((170, 260), dtype=torch.uint8, device=cuda_device)
    B1 = torch.zeros((170, 260), dtype=torch.uint8, device=cuda_device)
    B0[5:155, 11:211] = torch.from_numpy(I0).to(cuda_device)
    B1[5:155, 11:211] = torch.from_numpy(I1).to(cuda_device)
    F = torch.zeros((160, 230, 2), dtype=torch.float32, device=cuda_device)
    out = _alg(p).calc(B0[5:155, 11:211], B1[5:155, 11:211], F[3:153, 7:207])
    torch.cuda.synchronize()
    _assert_bits(out.cpu().numpy().copy(), M.calc(I0, I1, p))
    assert float(F[:3].abs().max()) == 0.0


def test_refusals(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200._lib import B2FError
    a = ocb.DISOpticalFlow_create(1)
    f32 = torch.zeros((64, 64), dtype=torch.float32, device=cuda_device)
    with pytest.raises(B2FError) as e:
        a.calc(f32, f32)
    assert e.value.status == 2
    u8 = torch.zeros((64, 64), dtype=torch.uint8, device=cuda_device)
    u8b = torch.zeros((64, 80), dtype=torch.uint8, device=cuda_device)
    with pytest.raises(B2FError) as e:
        a.calc(u8, u8b)
    assert e.value.status == 3
    b = ocb.DISOpticalFlow_create(1)
    b.setPatchSize(12)
    with pytest.raises(B2FError) as e:
        b.calc(u8, u8)
    assert e.value.status == 1


def test_determinism_and_streams(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    pairs = [synth.make_pair(240, 320, seed=20 + i, kind="smooth", mag=4.0)[:2] for i in range(4)]
    seq = [_run(cuda_device, a, b, None, ocb.DISOpticalFlow_create(1))[0] for a, b in pairs]
    again = _run(cuda_device, *pairs[0], None, ocb.DISOpticalFlow_create(1))[0]
    _assert_bits(again, seq[0])
    outs = [None] * 4

    def work(i):
        s = torch.cuda.Stream(device=cuda_device)
        alg = ocb.DISOpticalFlow_create(1)
        with torch.cuda.stream(s):
            d0, d1 = (torch.from_numpy(x).to(cuda_device) for x in pairs[i])
            for _ in range(2):  # the second call replays the graph
                f = alg.calc(d0, d1, stream=s)
        s.synchronize()
        outs[i] = f.cpu().numpy()

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for o, r in zip(outs, seq):
        _assert_bits(o, r)


def test_batch_and_default_stream(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200.batch import NativeFlowBatch
    I0, I1, _ = synth.make_pair(120, 160, seed=8, kind="smooth", mag=2.0)
    want = M.calc(I0, I1, M.DISParams())
    nb = NativeFlowBatch("dis", dict(), n_streams=2)
    out = [np.zeros((120, 160, 2), np.float32) for _ in range(3)]
    nb.run_host([(I0, I1)] * 3, out)
    nb.close()
    for o in out:
        _assert_bits(o, want)
    # the NULL stream: the call synchronises the device
    alg = ocb.DISOpticalFlow_create(1)
    f = alg.calc(torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device), stream=0)
    _assert_bits(f.cpu().numpy(), want)


@pytest.mark.parametrize("preset", [0, 1, 2])
def test_against_cv2_statistical(cuda_device, preset):
    """Propagation on: the engine's OpenCL-style propagation against cv2's CPU one, with the measured bounds and
    multiples of tests/test_dis_model_cpu.py (the engine equals the model bit for bit)."""
    import cv2
    I0, I1, gt = synth.make_pair(480, 640, seed=1, kind="smooth", mag=4.0)
    import opencv_contrib_b200 as ocb
    got, _ = _run(cuda_device, I0, I1, None, ocb.DISOpticalFlow_create(preset))
    ref = cv2.DISOpticalFlow_create(preset).calc(I0, I1, None)
    d = np.linalg.norm(got - ref, axis=-1)
    q50, q99 = M.CV2_MEASURED[preset]
    assert np.median(d) <= 2 * q50 and np.quantile(d, 0.99) <= 2 * q99 and d.max() <= 1.0
    e_got, e_ref = np.linalg.norm(got - gt, axis=-1).mean(), np.linalg.norm(ref - gt, axis=-1).mean()
    assert e_got <= 1.05 * e_ref + 0.005


def test_abi_symbols():
    from opencv_contrib_b200 import _lib
    l = _lib.lib()
    for name in ("b2f_dis_default_params", "b2f_dis_create"):
        assert hasattr(l, name)
    p = _lib.b2f_dis_params()
    l.b2f_dis_default_params(p, 2)
    assert (p.finest_scale, p.patch_stride, p.grad_descent_iterations, p.patch_size) == (1, 3, 25, 8)
