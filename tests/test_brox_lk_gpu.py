"""GPU tests for BroxOpticalFlow and DensePyrLKOpticalFlow (through the C ABI via ctypes).

Both algorithms are *parity unpinned* upstream (no CPU implementation; Brox's golden file lives in
opencv_extra, DensePyrLK has no accuracy test at all -- SURVEY.md §8c), so the engine is compared
with the numpy restatements of the CUDA reference (oracle/brox_model.py, oracle/denselk_model.py),
plus the reference's own sanity criteria: no NaN/Inf (BroxOpticalFlow.OpticalFlowNan,
test_optflow.cpp:130-161) and recovery of a known synthetic motion.
"""
import numpy as np
import pytest

from oracle import synth, brox_model as bm, brox_model_native as bmn, denselk_model as lk, denselk_model_native as lkn

pytestmark = pytest.mark.gpu


def _brox(dev, I0, I1, graph=1, aux=0, **kw):
    import torch
    import opencv_contrib_b200 as ocb
    alg = ocb.BroxOpticalFlow_create(**kw)
    alg.setEngineOption("use_graph", graph)
    alg.setEngineOption("aux_path", aux)
    f = alg.calc(torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev))
    torch.cuda.synchronize()
    return f.cpu().numpy(), alg


@pytest.mark.parametrize("h,w,kind", [(96, 128, "const"), (121, 163, "smooth")])
def test_brox_matches_model(cuda_device, h, w, kind):
    """With the data term's rsqrt correctly rounded (aux_path 1) the engine equals the model bit for bit; the C model
    equals the numpy statement.  The production rsqrtf (aux_path 0) is bounded by 4x the distance between the exact
    model and the model with the rsqrt moved by up to 2 ulp (tests/test_brox_fullsize_gpu.py)."""
    I0, I1, gt = synth.make_pair(h, w, seed=3, kind=kind, dtype="f32")
    kw = dict(alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=5, outer_iterations=77, solver_iterations=5)
    ref = bm.calc(I0, I1, bm.BroxParams(**kw))
    assert np.array_equal(bmn.calc(I0, I1, bm.BroxParams(**kw)).view(np.int32), ref.view(np.int32))
    for graph in (0, 1):
        got, alg = _brox(cuda_device, I0, I1, graph=graph, aux=1, **kw)
        assert np.isfinite(got).all()
        assert np.array_equal(got.view(np.int32), ref.view(np.int32)), (graph, int((got != ref).any(axis=-1).sum()))
    assert alg.getStats()["levels"] == len(bm.pyramid_sizes(h, w, 0.8, 77))
    assert alg.getDefaultName() == "DenseOpticalFlow.BroxOpticalFlow"
    got, _ = _brox(cuda_device, I0, I1, graph=1, **kw)
    pert = bmn.calc(I0, I1, bm.BroxParams(**kw), "perturbed")
    err, yard = np.abs(got - ref), np.abs(pert - ref)
    for q in (0.5, 0.99, 1.0):
        assert np.quantile(err, q) <= max(4 * np.quantile(yard, q), 1e-6), (q, float(np.quantile(err, q)),
                                                                              float(np.quantile(yard, q)))


@pytest.mark.parametrize("h,w,solver", [(150, 203, 7), (61, 64, 10), (300, 417, 10)])
def test_brox_fused_sor_bit_identical_to_half_sweep_kernels(cuda_device, h, w, solver):
    """kernel_path=1 runs one launch per red/black half sweep (the reference's shape); path 2 fuses up to 5
    iterations per launch in shared memory; the default path (0) keeps the cells in registers, one prepare + one solver
    launch per inner step; path 3 additionally runs ALL inner steps of a level in one cooperative launch (grid-wide barriers
    between the prepare and solver phases) wherever the level's regions are co-resident.  Same arithmetic, same order
    (brox_sor_cell) -> same bits, including levels that fit one region and odd sizes; inner = 3 and 4 cover both parities
    of the (du, dv) ping-pong."""
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(h, w, seed=7, kind="smooth", dtype="f32")
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    for inner in (3, 4):
        outs, launches = [], []
        for path in (0, 1, 2, 3):
            alg = ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, inner, 77, solver)
            alg.setEngineOption("kernel_path", path)
            outs.append(alg.calc(d0, d1).cpu().numpy())
            again = alg.calc(d0, d1).cpu().numpy()          # graph replay (barrier counter zeroed by its memset node)
            assert np.array_equal(again, outs[-1]), path
            launches.append(alg.getStats()["launches"])
        assert np.isfinite(outs[0]).all()
        assert np.array_equal(outs[0], outs[1]), (inner, float(np.abs(outs[0] - outs[1]).max()))
        assert np.array_equal(outs[2], outs[1]), (inner, float(np.abs(outs[2] - outs[1]).max()))
        assert np.array_equal(outs[3], outs[1]), (inner, float(np.abs(outs[3] - outs[1]).max()))
        assert launches[3] < launches[0], launches        # the cooperative level kernel replaced launches


def test_brox_reference_test_parameters_recover_motion(cuda_device):
    # the only parameter set the reference ever runs: create(0.197, 50, 0.8, 10, 77, 10) (test_optflow.cpp:75-76)
    I0, I1, gt = synth.make_pair(240, 320, seed=1, kind="const", dtype="f32")
    got, _ = _brox(cuda_device, I0, I1, alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=10,
                   outer_iterations=77, solver_iterations=10)
    assert np.isfinite(got).all()                        # OpticalFlowNan criterion
    c = got[24:-24, 24:-24]
    assert abs(float(np.median(c[..., 0])) - 2.5) < 0.15 and abs(float(np.median(c[..., 1])) + 1.25) < 0.15
    again, _ = _brox(cuda_device, I0, I1, alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=10,
                     outer_iterations=77, solver_iterations=10)
    assert np.array_equal(again, got)                    # deterministic


def test_brox_error_codes(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    a = torch.zeros((64, 64), dtype=torch.uint8, device=cuda_device)
    alg = ocb.BroxOpticalFlow_create()
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, a)
    assert e.value.status == 2                           # CV_32FC1 only (brox.cpp:134)
    alg = ocb.BroxOpticalFlow_create(alpha=0.0)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a.float(), a.float())
    assert e.value.status == 1                           # "Invalid alpha" (NCVBroxOpticalFlow.cu:606)


def _lk(dev, I0, I1, **kw):
    import torch
    import opencv_contrib_b200 as ocb
    alg = ocb.DensePyrLKOpticalFlow_create(**kw)
    f = alg.calc(torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev))
    torch.cuda.synchronize()
    return f.cpu().numpy(), alg


@pytest.mark.parametrize("win,levels,iters", [((7, 7), 2, 10), ((13, 13), 3, 30), ((5, 9), 1, 5)])
def test_denselk_matches_model(cuda_device, win, levels, iters):
    I0, I1, gt = synth.make_pair(72, 100, seed=5, kind="const")
    ref = lk.calc(I0, I1, win, levels, iters)
    assert np.array_equal(lkn.calc(I0, I1, win, levels, iters).view(np.int32), ref.view(np.int32))
    got, alg = _lk(cuda_device, I0, I1, winSize=win, maxLevel=levels, iters=iters)
    assert np.isfinite(got).all()
    # the model restates the kernels' roundings (FMA included), so the int-truncated samples agree exactly
    assert np.array_equal(got.view(np.int32), ref.view(np.int32)), int((got != ref).any(axis=-1).sum())
    assert alg.getDefaultName() == "DenseOpticalFlow.DensePyrLKOpticalFlow"
    assert alg.getWinSize() == win and alg.getMaxLevel() == levels and alg.getNumIters() == iters


def test_denselk_recovers_motion_and_rejects_bad_args(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, gt = synth.make_pair(240, 320, seed=2, kind="const")
    got, _ = _lk(cuda_device, I0, I1)                    # defaults 13x13, 3 levels, 30 iterations
    c = got[32:-32, 32:-32]
    assert abs(float(np.median(c[..., 0])) - 2.5) < 0.2 and abs(float(np.median(c[..., 1])) + 1.25) < 0.2
    again, _ = _lk(cuda_device, I0, I1)
    assert np.array_equal(again, got)
    a = torch.zeros((64, 64), dtype=torch.float32, device=cuda_device)
    with pytest.raises(ocb.B2FError) as e:
        ocb.DensePyrLKOpticalFlow_create().calc(a, a)
    assert e.value.status == 2                           # CV_8UC1 only (pyrlk.cpp:240)
    with pytest.raises(ocb.B2FError) as e:
        ocb.DensePyrLKOpticalFlow_create(winSize=(2, 13)).calc(a.to(torch.uint8), a.to(torch.uint8))
    assert e.value.status == 1                           # winSize > 2 (pyrlk.cpp:243)


@pytest.mark.parametrize("win_h,levels", [(13, 3), (7, 1)])
def test_denselk_fast_kernel_bit_identical_to_generic(cuda_device, win_h, levels):
    """Window width 13 takes the kernel that hoists the x half of every bilinear fetch into registers
    (kernel_path 0); kernel_path 1 forces the generic per-tap kernel.  Same arithmetic per tap."""
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(131, 177, seed=9, kind="smooth")
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    outs = []
    for path in (0, 1):
        alg = ocb.DensePyrLKOpticalFlow_create(winSize=(13, win_h), maxLevel=levels, iters=12)
        alg.setEngineOption("kernel_path", path)
        outs.append(alg.calc(d0, d1, torch.zeros((131, 177, 2), device=cuda_device)).cpu().numpy())
    assert np.array_equal(outs[0], outs[1]), float(np.abs(outs[0] - outs[1]).max())
