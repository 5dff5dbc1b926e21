"""GPU parity tests for FarnebackOpticalFlow (through the C ABI via ctypes).

Parity anchor: the LIVE CPU reference cv2.calcOpticalFlowFarneback (opencv/opencv modules/video,
the function modules/optflow/src/interfaces.cpp:154-157 forwards to), with the reference test's own
criteria (test_optflow.cpp:341-348): NCC dissimilarity <= 1e-4 (box) / 2e-2 (gaussian), plus a
mean-EPE bound, and committed golden fixtures (tests/golden/farneback_*.npz, made by
tests/golden/make_golden.py from cv2) so the check does not depend on the box's cv2.  Against the model of the
engine's own roundings (oracle/farneback_model.c) the comparison is exact.
"""
import os

import numpy as np
import cv2
import pytest

from oracle import synth, metrics, farneback_gpu_model as fm, farneback_model_native as fn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _run(dev, I0, I1, init=None, **kw):
    import torch
    import opencv_contrib_b200 as ocb
    alg = ocb.FarnebackOpticalFlow_create(**kw)
    d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
    fl = None if init is None else torch.from_numpy(init.copy()).to(dev)
    f = alg.calc(d0, d1, fl)
    torch.cuda.synchronize()
    return f.cpu().numpy(), alg


def _cv2(I0, I1, init=None, **kw):
    return cv2.calcOpticalFlowFarneback(I0, I1, None if init is None else init.copy(), kw.get("pyrScale", 0.5),
                                        kw.get("numLevels", 5), kw.get("winSize", 13), kw.get("numIters", 10),
                                        kw.get("polyN", 5), kw.get("polySigma", 1.1), kw.get("flags", 0))


CASES = [
    (dict(), 1e-4, 0.02),
    (dict(polyN=7, polySigma=1.5), 1e-4, 0.02),
    (dict(pyrScale=0.8, numLevels=3), 1e-4, 0.02),
    (dict(pyrScale=0.3, numLevels=3), 1e-4, 0.02),
    (dict(winSize=9, numIters=3), 1e-4, 0.02),
    (dict(flags=256), 2e-2, 0.2),
]


@pytest.mark.parametrize("kw,ncc_tol,epe_tol", CASES)
@pytest.mark.parametrize("h,w,kind,seed", [(240, 320, "smooth", 1), (243, 317, "affine", 2)])
def test_engine_vs_live_cpu_reference(cuda_device, kw, ncc_tol, epe_tol, h, w, kind, seed):
    I0, I1, _ = synth.make_pair(h, w, seed=seed, kind=kind)
    got, _ = _run(cuda_device, I0, I1, **kw)
    cpu = _cv2(I0, I1, **kw)
    assert np.isfinite(got).all()
    assert metrics.ncc_dissimilarity(got, cpu) <= ncc_tol
    assert metrics.epe_stats(got, cpu)["mean"] <= epe_tol


def _bits_equal(got, want):
    """got equals want bit for bit, NaN compared by position."""
    both_nan = np.isnan(got) & np.isnan(want)
    return bool(((got.view(np.uint32) == want.view(np.uint32)) | both_nan).all())


@pytest.mark.parametrize("kw", [dict(), dict(flags=256), dict(fastPyramids=True), dict(polyN=7, polySigma=1.5)])
def test_engine_matches_cuda_semantics_model(cuda_device, kw):
    """Bit for bit against the model of the engine's roundings (oracle/farneback_model.c, build "eng")."""
    I0, I1, _ = synth.make_pair(200, 264, seed=3, kind="smooth")
    got, _ = _run(cuda_device, I0, I1, **kw)
    P = fm.FarnebackParams(**kw)
    ref = fn.calc(I0, I1, P, build="eng", order=fn.order_for(P))
    assert _bits_equal(got, ref), metrics.epe_stats(got, ref)


def test_register_blocked_iteration_matches_generic_kernel(cuda_device):
    """kernel_path=1 forces the generic fused-iteration kernel (box window summed pair by pair, first gaussian tap
    rounded on its own); the K=6 register-blocked kernel runs the tree-plus-running box sum and fuses the first gaussian
    tap.  Each path equals the model in its own iteration order, bit for bit."""
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(203, 277, seed=4, kind="smooth")
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    for flags in (0, 256):
        P = fm.FarnebackParams(flags=flags)
        for path in (0, 1):
            alg = ocb.FarnebackOpticalFlow_create(flags=flags)
            alg.setEngineOption("kernel_path", path)
            got = alg.calc(d0, d1).cpu().numpy()
            ref = fn.calc(I0, I1, P, build="eng", order=fn.order_for(P, path))
            assert _bits_equal(got, ref), (flags, path, metrics.epe_stats(got, ref))


def test_golden_fixtures(cuda_device):
    names = sorted(n for n in os.listdir(GOLD) if n.startswith("farneback_") and n.endswith(".npz"))
    assert names, "golden fixtures missing"
    for n in names:
        z = np.load(os.path.join(GOLD, n))
        kw = {k[3:]: z[k].item() for k in z.files if k.startswith("kw_")}
        got, _ = _run(cuda_device, z["I0"], z["I1"], **kw)
        gold = z["flow"].astype(np.float32)
        assert metrics.ncc_dissimilarity(got, gold) <= float(z["ncc_tol"]), n
        assert metrics.epe_stats(got, gold)["mean"] <= float(z["epe_tol"]), n


def test_initial_flow_and_float_input(cuda_device):
    I0, I1, gt = synth.make_pair(240, 320, seed=3, kind="smooth")
    init = (gt + 0.3).astype(np.float32)
    got, _ = _run(cuda_device, I0, I1, init=init, flags=4)
    cpu = _cv2(I0, I1, init=init, flags=4)
    assert metrics.ncc_dissimilarity(got, cpu) <= 1e-4
    gotf, _ = _run(cuda_device, I0.astype(np.float32), I1.astype(np.float32))
    gotu, _ = _run(cuda_device, I0, I1)
    assert np.array_equal(gotf, gotu)   # no scaling on conversion (farneback.cpp:342-345)


def test_error_codes(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    a = torch.zeros((64, 64), dtype=torch.uint8, device=cuda_device)
    alg = ocb.FarnebackOpticalFlow_create(polyN=6)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, a)
    assert e.value.status == 1                                   # polyN in {5,7} (farneback.cpp:316)
    alg = ocb.FarnebackOpticalFlow_create(fastPyramids=True, pyrScale=0.8)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, a)
    assert e.value.status == 1                                   # fastPyramids => pyrScale 0.5 (:317)
    alg = ocb.FarnebackOpticalFlow_create()
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, torch.zeros((64, 80), dtype=torch.uint8, device=cuda_device))
    assert e.value.status == 3


def test_1080p_vs_live_cpu_reference(cuda_device):
    """BASELINE configs[1]: 1920x1080, 5 levels (perf config perf_optflow.cpp:242-258)."""
    I0, I1, gt = synth.make_pair(1080, 1920, seed=0, kind="smooth")
    got, alg = _run(cuda_device, I0, I1)
    cpu = _cv2(I0, I1)
    assert alg.getStats()["levels"] == 6
    assert metrics.ncc_dissimilarity(got, cpu) <= 1e-4
    assert metrics.epe_stats(got, cpu)["mean"] <= 0.02
    again, _ = _run(cuda_device, I0, I1)
    assert np.array_equal(again, got)


@pytest.mark.parametrize("flags", [0, 256])
def test_persistent_tma_iteration_kernel_bit_identical(cuda_device, flags):
    """kernel_path = 3: levels with at least two waves of 64x64 tiles run the persistent kernel whose M tiles arrive
    by TMA (zero fill patched to replicate borders).  Same arithmetic -> same bits, including ragged borders."""
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(1030, 1290, seed=3, kind="smooth")
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    outs = []
    for path in (0, 3):
        alg = ocb.FarnebackOpticalFlow_create(numLevels=2, numIters=3, flags=flags)
        alg.setEngineOption("kernel_path", path)
        outs.append(alg.calc(d0, d1).cpu().numpy())
    assert np.isfinite(outs[1]).all()
    assert np.array_equal(outs[0], outs[1]), float(np.abs(outs[0] - outs[1]).max())


def test_iteration_kernel_register_variants_bit_identical(cuda_device):
    """aux_path picks the register cap (= resident blocks per SM) of the fused iteration kernel: 0 -> 128 registers
    (default), 3 -> 80, 4 -> 64, 5 -> the lane-transposed R1 gather.  They run on levels with more than n_SM 64x32 tiles
    (smaller levels take the 512-thread kernel), so level 0 is sized from the SM count.  Same arithmetic -> same bits."""
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200._lib import FARN_PATH
    n_sm = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    h, w = 32 * (n_sm // 15 + 2) - 5, 960 - 27   # 15 x (n_SM / 15 + 2) > n_SM tiles at level 0, about a quarter at level 1
    I0, I1, _ = synth.make_pair(h, w, seed=13, kind="smooth")
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    outs = []
    for aux, path in ((0, "quad"), (3, "quad_r80"), (4, "quad_r64"), (5, "quad_transposed")):
        alg = ocb.FarnebackOpticalFlow_create()
        alg.setEngineOption("aux_path", aux)
        outs.append(alg.calc(d0, d1).cpu().numpy())
        levels = alg.getStats()["levels"]
        assert [alg.getActivePath(k) for k in range(levels)] == [FARN_PATH[path]] + [FARN_PATH["quad_wide"]] * (levels - 1)
    for o in outs[1:]:
        assert np.array_equal(outs[0], o)


@pytest.mark.parametrize("h,w", [(270, 480), (203, 277)])
@pytest.mark.parametrize("poly_n,sigma", [(5, 1.1), (7, 1.5)])
def test_polyexp_register_blocked_kernel_bit_identical(cuda_device, h, w, poly_n, sigma):
    """The default secondary kernels -- polynomial expansion on 64x32 blocks (vertical pass from a register window, float4
    horizontal pass) and the sparse vertical blur with four columns per thread -- against the round-1 kernels (aux_path 6):
    same expressions in the same order -> same flow bits, including ragged right / bottom blocks, levels smaller than one
    block, and non-integral pyramid scales."""
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(h, w, seed=17, kind="smooth")
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    # pyrScale 0.5: integral 1 / scale (only the even rows of the sparse vertical blur are launched); 0.8: both bilinear rows
    for pyr_scale, levels in ((0.5, 5), (0.8, 4)):
        outs = []
        for aux in (0, 6):
            alg = ocb.FarnebackOpticalFlow_create(numLevels=levels, pyrScale=pyr_scale, polyN=poly_n, polySigma=sigma)
            alg.setEngineOption("aux_path", aux)
            outs.append(alg.calc(d0, d1).cpu().numpy())
        assert np.isfinite(outs[0]).all()
        assert np.array_equal(outs[0], outs[1]), (pyr_scale, float(np.abs(outs[0] - outs[1]).max()))
