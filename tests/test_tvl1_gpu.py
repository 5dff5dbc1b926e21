"""GPU parity tests for OpticalFlowDual_TVL1 (through the C ABI via ctypes).

Tolerances (stated -- see DESIGN.md "Parity"):
  * engine vs the CUDA-semantics numpy model: max |dflow| <= 1e-3 px (gamma = 0);
  * engine vs the CPU reference oracle (modules/optflow semantics): >= 95 % of interior pixels
    with EPE <= 0.1 px, mean EPE <= 0.08 px, NCC dissimilarity <= 4e-3
    (reference criteria: test_tvl1optflow.cpp:114-142, test_optflow.cpp:462-465);
  * temporally blocked kernel vs unfused kernels: bit-identical;
  * concurrent instances on separate streams vs synchronous: bit-identical (test_optflow.cpp:468-528).
"""
import threading

import numpy as np
import pytest

from oracle import synth, metrics, tvl1_cpu, tvl1_gpu_model as gm

pytestmark = pytest.mark.gpu


def _run(dev, I0, I1, path=0, fused=0, graph=1, stream=None, init=None, _median=None, aux=0, **kw):
    import torch
    import opencv_contrib_b200 as ocb
    alg = ocb.OpticalFlowDual_TVL1_create(**kw)
    alg.setEngineOption("aux_path", aux)
    if _median is not None:
        alg.setMedianFiltering(_median[0])
        alg.setMedianPeriod(_median[1])
    alg.setEngineOption("kernel_path", path)
    alg.setEngineOption("fused_iters", fused)
    alg.setEngineOption("use_graph", graph)
    d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
    fl = None if init is None else torch.from_numpy(init.copy()).to(dev)
    f = alg.calc(d0, d1, fl, stream)
    torch.cuda.synchronize()
    return f.cpu().numpy(), alg


@pytest.mark.parametrize("h,w,kind,seed", [(120, 160, "const", 0), (243, 317, "smooth", 1), (97, 131, "affine", 2)])
def test_engine_matches_cuda_semantics_model(cuda_device, h, w, kind, seed):
    I0, I1, gt = synth.make_pair(h, w, seed=seed, kind=kind)
    kw = dict(nscales=4, warps=3, epsilon=0.0, iterations=20)
    ref = gm.calc(I0, I1, gm.TVL1Params(**kw))
    for path in (1, 2, 0):
        got, alg = _run(cuda_device, I0, I1, path=path, **kw)
        st = metrics.epe_stats(got, ref)
        assert np.isfinite(got).all() and st["max"] <= 1e-3, (path, st)
    assert alg.getStats()["launches"] > 0
    for aux in (3,):                                       # separable warp kernel on every level
        alt, _ = _run(cuda_device, I0, I1, aux=aux, **kw)
        st = metrics.epe_stats(alt, ref)
        assert np.isfinite(alt).all() and st["max"] <= 1e-3, ("warp kernel variant", aux, st)


@pytest.mark.parametrize("K", [1, 2, 3, 5, 6, 7, 10, 12])
def test_blocked_kernel_bit_identical_to_unfused(cuda_device, K):
    # odd sizes: tiles straddle every image border
    I0, I1, _ = synth.make_pair(203, 277, seed=3, kind="smooth")
    kw = dict(nscales=3, warps=2, epsilon=0.0, iterations=23)
    a, _ = _run(cuda_device, I0, I1, path=1, **kw)
    # 0 = persistent TMA kernel, 2 = blocked kernel with plain loads
    for path in (0, 2):
        for graph in (0, 1):
            b, _ = _run(cuda_device, I0, I1, path=path, fused=K, graph=graph, **kw)
            assert np.array_equal(a, b), (path, K, graph, float(np.abs(a - b).max()))


def test_engine_vs_cpu_reference_oracle_epe(cuda_device):
    # parameter mapping of the reference's own GPU-vs-CPU test (test_optflow.cpp:448-460)
    I0, I1, gt = synth.make_pair(240, 320, seed=4, kind="smooth")
    got, _ = _run(cuda_device, I0, I1, nscales=5, warps=5, epsilon=0.0, iterations=30)
    cpu = tvl1_cpu.calc(I0, I1, tvl1_cpu.TVL1Params(nscales=5, warps=5, epsilon=0.0, innerIterations=1,
                                                    outerIterations=30, medianFiltering=1))
    st = metrics.epe_stats(got, cpu, border=16)
    ncc = metrics.ncc_dissimilarity(got[16:-16, 16:-16], cpu[16:-16, 16:-16])
    assert st["frac_le_0.1"] >= 0.95 and st["mean"] <= 0.08 and ncc <= 4e-3, (st, ncc)


def test_default_epsilon_cadence_matches_model(cuda_device):
    I0, I1, _ = synth.make_pair(120, 160, seed=2, kind="const")
    kw = dict(nscales=3, warps=3, epsilon=0.01, iterations=100)
    tr = []
    ref = gm.calc(I0, I1, gm.TVL1Params(**kw), trace=tr)
    got, alg = _run(cuda_device, I0, I1, **kw)
    assert metrics.epe_stats(got, ref)["max"] <= 1e-3
    assert alg.getStats()["iterations_run"] == sum(sum(t) for t in tr)


def test_device_side_convergence_loop_equals_host_loop(cuda_device):
    """epsilon > 0 on a real stream: the reference's adaptive stopping rule runs as a WHILE conditional node of the CUDA
    graph (no host synchronisation inside calc); on the legacy default stream / without a graph the host decides like
    the reference does (tvl1flow.cpp:357-380).  Same cadence, same arithmetic -> same bits, same iteration count."""
    import torch
    I0, I1, _ = synth.make_pair(150, 190, seed=6, kind="smooth")
    for kw in (dict(nscales=3, warps=3, epsilon=0.01, iterations=100), dict(nscales=2, warps=2, epsilon=0.05, iterations=37),
               dict()):  # the reference's create() defaults
        host, a_host = _run(cuda_device, I0, I1, graph=0, **kw)
        side = torch.cuda.Stream(device=cuda_device)
        dev, a_dev = _run(cuda_device, I0, I1, graph=1, stream=side, **kw)
        assert np.array_equal(host, dev), float(np.abs(host - dev).max())
        assert a_dev.getStats()["iterations_run"] == a_host.getStats()["iterations_run"] > 0
        again, _ = _run(cuda_device, I0, I1, graph=1, stream=side, **kw)
        assert np.array_equal(again, dev)


def test_gamma_illumination_path(cuda_device):
    # gamma != 0 is chaotic (1e-7 input noise moves the model by ~0.1 px at a few pixels), so the
    # tolerance is statistical
    I0, I1, _ = synth.make_pair(120, 160, seed=2, kind="const")
    kw = dict(nscales=3, warps=3, epsilon=0.0, iterations=20, gamma=1.0)
    ref = gm.calc(I0, I1, gm.TVL1Params(**kw))
    got, _ = _run(cuda_device, I0, I1, **kw)
    st = metrics.epe_stats(got, ref)
    assert st["mean"] <= 5e-3 and st["frac_le_0.1"] >= 0.99, st


def test_float_input_and_initial_flow(cuda_device):
    I0, I1, gt = synth.make_pair(120, 160, seed=5, kind="const", dtype="f32")
    kw = dict(nscales=3, warps=3, epsilon=0.0, iterations=20)
    ref = gm.calc(I0, I1, gm.TVL1Params(**kw))
    got, _ = _run(cuda_device, I0, I1, **kw)
    assert metrics.epe_stats(got, ref)["max"] <= 1e-3
    init = (gt + 0.25).astype(np.float32)
    kw["useInitialFlow"] = True
    ref = gm.calc(I0, I1, gm.TVL1Params(**kw), init_flow=init)
    got, _ = _run(cuda_device, I0, I1, init=init, **kw)
    assert metrics.epe_stats(got, ref)["max"] <= 1e-3


def test_tiled_warp_kernel_bit_identical_to_separable(cuda_device):
    """The default warp kernel (aux_path 0) stages the I1 window of a 64x32 tile in shared memory (TMA) and gathers the
    taps from there; pixels whose window leaves the staged box (flow > 9 px) take the global-memory window, border pixels
    the clamped tap loop.  Same arithmetic as the separable kernel (aux_path 3): same bits, whatever path a pixel takes."""
    # pyramid: levels below 88x56 fall back to the separable kernel, the others tile with ragged right / bottom edges
    I0, I1, gt = synth.make_pair(203, 277, seed=3, kind="smooth")
    kw = dict(nscales=3, warps=3, epsilon=0.0, iterations=9)
    a, _ = _run(cuda_device, I0, I1, aux=3, **kw)
    b, alg = _run(cuda_device, I0, I1, aux=0, **kw)
    assert np.array_equal(a, b), float(np.abs(a - b).max())
    assert alg.getStats()["launches"] > 0
    # one level, initial flows from sub-pixel to far beyond the staged margin (and pointing out of the image)
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:203, 0:277].astype(np.float32)
    for amp in (0.7, 6.0, 11.5, 40.0):
        init = np.stack([amp * np.sin(xx / 37.0 + yy / 53.0), amp * np.cos(xx / 41.0 - yy / 29.0)], axis=-1).astype(np.float32)
        init += rng.uniform(-0.5, 0.5, init.shape).astype(np.float32)
        k1 = dict(nscales=1, warps=2, epsilon=0.0, iterations=5, useInitialFlow=True)
        a, _ = _run(cuda_device, I0, I1, aux=3, init=init, **k1)
        b, _ = _run(cuda_device, I0, I1, aux=0, init=init, **k1)
        assert np.isfinite(b).all() and np.array_equal(a, b), (amp, float(np.abs(a - b).max()))


def test_pitched_roi_inputs(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(100, 140, seed=6, kind="const")
    kw = dict(nscales=3, warps=2, epsilon=0.0, iterations=10)
    a, _ = _run(cuda_device, I0, I1, **kw)
    big0 = torch.zeros((128, 200), dtype=torch.uint8, device=cuda_device)
    big1 = torch.zeros((128, 200), dtype=torch.uint8, device=cuda_device)
    bigf = torch.zeros((128, 200, 2), dtype=torch.float32, device=cuda_device)
    big0[7:107, 13:153] = torch.from_numpy(I0).to(cuda_device)
    big1[7:107, 13:153] = torch.from_numpy(I1).to(cuda_device)
    alg = ocb.OpticalFlowDual_TVL1_create(**kw)
    alg.calc(big0[7:107, 13:153], big1[7:107, 13:153], bigf[7:107, 13:153])
    torch.cuda.synchronize()
    assert np.array_equal(bigf[7:107, 13:153].cpu().numpy(), a)
    assert float(bigf[:7].abs().max()) == 0.0 and float(bigf[:, :13].abs().max()) == 0.0


def test_concurrent_streams_bit_identical(cuda_device):
    # reference: OpticalFlowDual_TVL1.Async (test_optflow.cpp:468-528)
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(160, 200, seed=7, kind="smooth")
    kw = dict(nscales=3, warps=3, epsilon=0.0, iterations=20)
    gold, _ = _run(cuda_device, I0, I1, **kw)
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    n = 8
    algs = [ocb.OpticalFlowDual_TVL1_create(**kw) for _ in range(n)]
    streams = [torch.cuda.Stream(device=cuda_device) for _ in range(n)]
    outs = [None] * n

    def work(i):
        outs[i] = algs[i].calc(d0, d1, None, streams[i])

    th = [threading.Thread(target=work, args=(i,)) for i in range(n)]
    [t.start() for t in th]
    [t.join() for t in th]
    torch.cuda.synchronize()
    for o in outs:
        assert np.array_equal(o.cpu().numpy(), gold)


def test_stream_ordering_after_prior_work(cuda_device):
    # reference: FarnebackOpticalFlowAsync (test_optflow.cpp:359-416): work enqueued on the caller's
    # stream before calc must be visible to it
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(160, 200, seed=8, kind="const")
    kw = dict(nscales=3, warps=2, epsilon=0.0, iterations=10)
    gold, _ = _run(cuda_device, I0, I1, **kw)
    s = torch.cuda.Stream(device=cuda_device)
    h0, h1 = torch.from_numpy(I0).pin_memory(), torch.from_numpy(I1).pin_memory()
    dummy = torch.empty(48 << 20, dtype=torch.uint8).pin_memory()
    alg = ocb.OpticalFlowDual_TVL1_create(**kw)
    with torch.cuda.stream(s):
        big = dummy.to(cuda_device, non_blocking=True)
        d0 = h0.to(cuda_device, non_blocking=True)
        d1 = h1.to(cuda_device, non_blocking=True)
        out = alg.calc(d0, d1, None, s)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), gold) and big.numel() > 0


def test_host_buffer_entry_point(cuda_device):
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(120, 160, seed=9, kind="const")
    kw = dict(nscales=3, warps=2, epsilon=0.0, iterations=10)
    gold, _ = _run(cuda_device, I0, I1, **kw)
    alg = ocb.OpticalFlowDual_TVL1_create(**kw)
    assert np.array_equal(alg.calc_host(I0, I1), gold)


def test_error_codes(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    alg = ocb.OpticalFlowDual_TVL1_create()
    a = torch.zeros((64, 64), dtype=torch.uint8, device=cuda_device)
    b = torch.zeros((64, 65), dtype=torch.uint8, device=cuda_device)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, b)
    assert e.value.status == 3                                    # size mismatch (tvl1flow.cpp:188)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, a.float())
    assert e.value.status == 2                                    # type mismatch (tvl1flow.cpp:189)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a.to(torch.int16), a.to(torch.int16))
    assert e.value.status == 2                                    # only 8UC1 / 32FC1 (tvl1flow.cpp:187)
    alg.setNumScales(0)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, a)
    assert e.value.status == 1                                    # nscales > 0 (tvl1flow.cpp:191)
    alg = ocb.OpticalFlowDual_TVL1_create(useInitialFlow=True)
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(a, a)                                            # initial flow requested but none supplied (:190)
    assert e.value.status == 1
    with pytest.raises(ocb.B2FError) as e:                        # short host pitch is a bad argument, not a CUDA error
        import ctypes as C
        from opencv_contrib_b200 import _lib
        h = np.zeros((64, 64), np.uint8)
        f = np.zeros((64, 64, 2), np.float32)
        i0 = _lib.b2f_image(h.ctypes.data, 32, 64, 64, 0)
        fl = _lib.b2f_image(f.ctypes.data, 512, 64, 64, 13)
        st = _lib.lib().b2f_calc_host(ocb.OpticalFlowDual_TVL1_create()._h, C.byref(i0), C.byref(i0), C.byref(fl), None)
        raise ocb.B2FError(st)
    assert e.value.status == 1


def test_1080p_round_trip_properties(cuda_device):
    """Full BASELINE size: size-independent checks (the numpy oracles would take minutes)."""
    import torch
    I0, I1, gt = synth.make_pair(1080, 1920, seed=0, kind="const")
    kw = dict(nscales=5, warps=10, epsilon=0.0, iterations=30)
    got, alg = _run(cuda_device, I0, I1, **kw)
    assert np.isfinite(got).all() and alg.getStats()["levels"] == 5
    st = metrics.epe_stats(got, gt, border=32)          # recovers the known translation
    assert st["frac_le_0.1"] >= 0.95, st
    z, _ = _run(cuda_device, I0, I0, **kw)              # identical frames -> zero flow
    assert float(np.abs(z).max()) <= 1e-3
    again, _ = _run(cuda_device, I0, I1, **kw)          # run-to-run determinism
    assert np.array_equal(again, got)


def _cpu_reference(I0, I1, P):
    """The reference's own CPU source (oracle/_ref, built where an opencv_contrib tree is available) when present,
    else its bit-identical C port (tests/test_oracle_cpu.py pins the port to the reference's stored outputs)."""
    from oracle import tvl1_cpu_native, tvl1_ref
    if tvl1_ref.available():
        return tvl1_ref.calc(I0, I1, P), "reference"
    if tvl1_cpu_native.available():
        return tvl1_cpu_native.calc(I0, I1, P), "port"
    pytest.skip("neither oracle/_ref/libtvl1_ref.so nor oracle/_build/libtvl1_cpu.so is built")


def test_engine_vs_golden_reference_vectors(cuda_device):
    """tests/golden/tvl1_ref_*.npz: outputs of the reference's own modules/optflow/src/tvl1flow.cpp (compiled
    unmodified, make_golden.py).  GPU parameters are the twin the reference's GPU-vs-CPU test uses
    (test_optflow.cpp:456-460: iterations = inner * outer with inner = 1 ... here inner * outer in general);
    acceptance = that test's NCC bound plus the CPU regression criterion (>= 95 % within 0.1 px)."""
    import os
    gold = os.path.join(os.path.dirname(__file__), "golden")
    n = 0
    for name in sorted(os.listdir(gold)):
        if not (name.startswith("tvl1_ref_") and name.endswith(".npz")):
            continue
        z = np.load(os.path.join(gold, name))
        kw = {k[3:]: z[k].item() for k in z.files if k.startswith("kw_")}
        P = tvl1_cpu.TVL1Params(**kw)
        if P.epsilon > 0:
            continue                  # the CUDA path samples its stopping rule on another cadence (tvl1flow.cpp:357-380)
        n += 1
        got, _ = _run(cuda_device, z["I0"], z["I1"], nscales=P.nscales, warps=P.warps, epsilon=0.0,
                      iterations=P.innerIterations * P.outerIterations, gamma=P.gamma,
                      _median=(P.medianFiltering, P.innerIterations))
        st = metrics.epe_stats(got, z["flow"], border=16)
        ncc = metrics.ncc_dissimilarity(got[16:-16, 16:-16], z["flow"][16:-16, 16:-16])
        assert st["frac_le_0.1"] >= 0.95 and st["mean"] <= 0.08 and ncc <= 4e-3, (name, st, ncc)
    assert n >= 3


def test_median_filtering_knob_and_initial_flow_source(cuda_device):
    """MEDIAN_FILTERING / MEDIAN_PERIOD (the CPU / OpenCL class's medianFiltering, tvl1flow.cpp:1377-1383): a pass with
    kernel 5 must change the result, kernel 1 must not, the median kernel itself is the exact cv2.medianBlur; and
    INITIAL_FLOW_SOURCE 1 (the reference CUDA class's de-facto behaviour) equals feeding the previous result back."""
    import cv2
    import torch
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(120, 160, seed=3, kind="smooth")
    kw = dict(nscales=1, warps=1, epsilon=0.0, iterations=4)
    base, _ = _run(cuda_device, I0, I1, **kw)
    same, _ = _run(cuda_device, I0, I1, _median=(1, 2), **kw)
    med, _ = _run(cuda_device, I0, I1, _median=(5, 2), **kw)
    assert np.array_equal(base, same) and not np.array_equal(base, med)
    # the primitive itself is the exact cv2.medianBlur (pitched planes)
    import ctypes as C
    from opencv_contrib_b200 import _lib
    from opencv_contrib_b200.cudaoptflow import _image_from_tensor
    a = np.random.default_rng(0).normal(0, 2, (97, 131)).astype(np.float32)
    src = torch.zeros((97, 160), device=cuda_device)
    src[:, :131] = torch.from_numpy(a).to(cuda_device)
    for k in (3, 5):
        dst = torch.zeros((97, 131), device=cuda_device)
        si, di = _image_from_tensor(src[:, :131]), _image_from_tensor(dst)
        assert _lib.lib().b2f_median_blur_32f(C.byref(si), C.byref(di), k, None) == 0
        assert np.array_equal(dst.cpu().numpy(), cv2.medianBlur(a, k)), k
    # initial-flow source 1: second call starts from the first call's result
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    alg = ocb.OpticalFlowDual_TVL1_create(nscales=1, warps=2, epsilon=0.0, iterations=10, useInitialFlow=True)
    alg.setInitialFlowSource(1)
    first = alg.calc(d0, d1).cpu().numpy()                       # fresh handle: starts from zero
    second = alg.calc(d0, d1).cpu().numpy()
    ref0, _ = _run(cuda_device, I0, I1, nscales=1, warps=2, epsilon=0.0, iterations=10)
    ref1, _ = _run(cuda_device, I0, I1, init=ref0, nscales=1, warps=2, epsilon=0.0, iterations=10, useInitialFlow=True)
    assert np.array_equal(first, ref0) and np.array_equal(second, ref1)


def test_4k_baseline_config_vs_cpu_oracle(cuda_device):
    """BASELINE configs[4] frame size: 3840x2160, 5 scales / 10 warps / 30 iterations, eps = 0, one pair, against the
    CPU reference (same tolerances as the 1080p test).  Levels 3840x2160 ... 1573x885 (SURVEY.md §8)."""
    I0, I1, gt = synth.make_pair(2160, 3840, seed=0, kind="smooth")
    got, alg = _run(cuda_device, I0, I1, nscales=5, warps=10, epsilon=0.0, iterations=30)
    assert alg.getStats()["levels"] == 5 and np.isfinite(got).all()
    cpu, kind = _cpu_reference(I0, I1, tvl1_cpu.TVL1Params(nscales=5, warps=10, epsilon=0.0, innerIterations=1,
                                                           outerIterations=30, medianFiltering=1))
    st = metrics.epe_stats(got, cpu, border=32)
    ncc = metrics.ncc_dissimilarity(got[32:-32, 32:-32], cpu[32:-32, 32:-32])
    assert st["frac_le_0.1"] >= 0.95 and st["mean"] <= 0.08 and ncc <= 4e-3, (kind, st, ncc)
    g_gpu, g_cpu = metrics.epe_stats(got, gt, border=32), metrics.epe_stats(cpu, gt, border=32)
    assert abs(g_gpu["mean"] - g_cpu["mean"]) <= 0.05, (g_gpu, g_cpu)


def test_1080p_baseline_config_vs_cpu_oracle(cuda_device):
    """BASELINE configs[2] at full size: 1920x1080, 5 scales / 10 warps / 30 iterations, eps = 0, against the CPU
    oracle (the C/OpenMP port of modules/optflow/src/tvl1flow.cpp; a few seconds on the box's cores) at the
    reference's own GPU-vs-CPU acceptance level (test_optflow.cpp:456-465: NCC similarity; plus the regression
    criterion of test_tvl1optflow.cpp:114-142, >= 95 % of the pixels within 0.1 px)."""
    I0, I1, gt = synth.make_pair(1080, 1920, seed=0, kind="smooth")
    got, _ = _run(cuda_device, I0, I1, nscales=5, warps=10, epsilon=0.0, iterations=30)
    cpu, _kind = _cpu_reference(I0, I1, tvl1_cpu.TVL1Params(nscales=5, warps=10, epsilon=0.0, innerIterations=1,
                                                            outerIterations=30, medianFiltering=1))
    st = metrics.epe_stats(got, cpu, border=32)
    ncc = metrics.ncc_dissimilarity(got[32:-32, 32:-32], cpu[32:-32, 32:-32])
    assert st["frac_le_0.1"] >= 0.95 and st["mean"] <= 0.08 and ncc <= 4e-3, (st, ncc)
    # and both recover the synthetic motion equally well
    g_gpu, g_cpu = metrics.epe_stats(got, gt, border=32), metrics.epe_stats(cpu, gt, border=32)
    assert abs(g_gpu["mean"] - g_cpu["mean"]) <= 0.05, (g_gpu, g_cpu)
