"""GPU tests for the components either side of calc() (SURVEY.md 8f): planar output, interpolateFrames
argument checks (its model comparisons are in test_frames_gpu.py) and the video front end -- all through the
C ABI (ctypes).
"""
import numpy as np
import pytest

from oracle import synth, metrics

pytestmark = pytest.mark.gpu


def _algs(ocb):
    return {
        "tvl1": (lambda: ocb.OpticalFlowDual_TVL1_create(0.25, 0.15, 0.3, 3, 3, 0.0, 10, 0.8, 0.0, False), "u8"),
        "farneback": (lambda: ocb.FarnebackOpticalFlow_create(3, 0.5, False, 13, 3, 5, 1.1, 0), "u8"),
        "brox": (lambda: ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 3), "f32"),
        "denselk": (lambda: ocb.DensePyrLKOpticalFlow_create((7, 7), 2, 5, False), "u8"),
    }


@pytest.mark.parametrize("name", ["tvl1", "farneback", "brox", "denselk"])
def test_calc_uv_equals_split_of_calc(cuda_device, name):
    import torch
    import opencv_contrib_b200 as ocb
    make, dt = _algs(ocb)[name]
    I0, I1, _ = synth.make_pair(90, 131, seed=4, kind="smooth", dtype=dt)
    d0, d1 = torch.from_numpy(I0).to(cuda_device), torch.from_numpy(I1).to(cuda_device)
    alg = make()
    flow = alg.calc(d0, d1).cpu().numpy()
    # pitched planar outputs (ROI of wider buffers)
    u0 = torch.empty((90, 160), device=cuda_device)[:, 7:138]
    v0 = torch.empty((90, 192), device=cuda_device)[:, 1:132]
    u, v = alg.calcUV(d0, d1, u0, v0)
    torch.cuda.synchronize()
    assert np.array_equal(u.cpu().numpy(), flow[..., 0]) and np.array_equal(v.cpu().numpy(), flow[..., 1])
    with pytest.raises(ocb.B2FError):
        alg.calcUV(d0, d1, torch.empty((90, 131, 2), device=cuda_device)[..., 0].contiguous().to(torch.float64), v0)


def test_interpolate_frames_argument_checks(cuda_device):
    import torch
    import opencv_contrib_b200 as ocb
    z = torch.zeros((16, 32), device=cuda_device)
    with pytest.raises(ocb.B2FError):  # CV_Assert(frame0.type() == CV_32FC1)
        ocb.interpolateFrames(z.to(torch.uint8), z, z, z, z, z, 0.5)
    with pytest.raises(ocb.B2FError):  # size mismatch
        ocb.interpolateFrames(z, torch.zeros((16, 31), device=cuda_device), z, z, z, z, 0.5)
    with pytest.raises(ocb.B2FError):  # equal steps are required (interpolate_frames.cpp:82)
        ocb.interpolateFrames(z, torch.zeros((16, 64), device=cuda_device)[:, :32], z, z, z, z, 0.5)
    # zero flow, corrected: a plain cross-fade
    f0, f1 = torch.rand((16, 32), device=cuda_device), torch.rand((16, 32), device=cuda_device)
    out = ocb.interpolateFrames(f0, f1, z, z, z, z, 0.25, corrected=True)
    assert torch.allclose(out, 0.75 * f0 + 0.25 * f1, atol=1e-6)


def _frames(n, h, w, dt="u8"):
    """n frames of one texture translating by (1.5, -0.75) px per frame."""
    import cv2
    T = synth.texture(h + 64, w + 64, 11)
    out = []
    for k in range(n):
        M = np.float32([[1, 0, -32 + 1.5 * k], [0, 1, -32 - 0.75 * k]])
        f = cv2.warpAffine(T, M, (w, h), flags=cv2.INTER_CUBIC | cv2.WARP_INVERSE_MAP)
        f = np.clip(f, 0, 255)
        out.append(f.astype(np.uint8) if dt == "u8" else (f / 255).astype(np.float32))
    return out


@pytest.mark.parametrize("name,depth", [("tvl1", 1), ("tvl1", 3), ("farneback", 2), ("brox", 2)])
def test_video_front_end_equals_pairwise_calc(cuda_device, name, depth):
    import opencv_contrib_b200 as ocb
    make, dt = _algs(ocb)[name]
    frames = _frames(6, 120, 168, dt)
    ref_alg = make()
    want = [ref_alg.calc_host(frames[k], frames[k + 1]) for k in range(5)]
    vf = ocb.VideoFlow(make(), 120, 168, dtype=frames[0].dtype, depth=depth)
    got = dict(vf.run(frames))
    assert sorted(got) == list(range(5))
    for k in range(5):
        assert np.array_equal(got[k], want[k]), (k, float(np.abs(got[k] - want[k]).max()))
    # a pair that has left the ring can no longer be fetched
    with pytest.raises(ocb.B2FError):
        vf.fetch(0 if depth < 5 else 99)
    vf.close()


@pytest.mark.parametrize("name", ["tvl1", "farneback"])
def test_video_warm_start_chains_the_previous_flow(cuda_device, name):
    import opencv_contrib_b200 as ocb
    make, dt = _algs(ocb)[name]
    frames = _frames(5, 120, 168, dt)
    # by hand, as the reference test does (test_optflow.cpp:328-334): pair k starts from flow k-1
    alg = make()
    flow = alg.calc_host(frames[0], frames[1])
    want = [flow.copy()]
    if name == "tvl1":
        alg.setUseInitialFlow(True)
    else:
        alg.setFlags(ocb.OPTFLOW_USE_INITIAL_FLOW)
    for k in range(1, 4):
        flow = alg.calc_host(frames[k], frames[k + 1], flow.copy())
        want.append(flow.copy())
    for depth in (1, 2):
        host_alg = make()
        vf = ocb.VideoFlow(host_alg, 120, 168, dtype=frames[0].dtype, depth=depth, warm_start=True)
        got = dict(vf.run(frames))
        for k in range(4):
            assert np.array_equal(got[k], want[k]), (depth, k)
        vf.close()
        # the front end restores the algorithm's own setting
        assert (host_alg.getUseInitialFlow() if name == "tvl1" else host_alg.getFlags()) in (False, 0)
    # the chained solution still recovers the motion
    gt = np.zeros((120, 168, 2), np.float32)
    gt[..., 0], gt[..., 1] = -1.5, 0.75
    st = metrics.epe_stats(want[-1][16:-16, 16:-16], gt[16:-16, 16:-16])
    assert st["mean"] < 0.5, st
    with pytest.raises(ocb.B2FError):  # Brox has no initial-flow path
        ocb.VideoFlow(_algs(ocb)["brox"][0](), 120, 168, dtype=np.float32, warm_start=True)


def test_entry_points_follow_the_stream_device_not_the_thread_device(cuda_device):
    """The CUDA current device is per host thread; a worker thread that never called cudaSetDevice sits on
    device 0.  Every entry point switches to the device that owns the stream / the images for the call."""
    import threading
    import torch
    import opencv_contrib_b200 as ocb
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    d1 = torch.device("cuda:1")
    I0, I1, _ = synth.make_pair(96, 128, seed=2, kind="const")
    ref = ocb.FarnebackOpticalFlow_create(numLevels=3).calc_host(I0, I1)  # device 0, main thread
    out = {}

    def work():
        try:
            assert torch.cuda.current_device() == 0
            s = torch.cuda.Stream(device=d1)
            alg = ocb.FarnebackOpticalFlow_create(numLevels=3)
            out["host"] = alg.calc_host(I0, I1, None, s)
            a, b = torch.from_numpy(I0).to(d1), torch.from_numpy(I1).to(d1)
            f = alg.calc(a, b, torch.empty((96, 128, 2), device=d1), s)
            s.synchronize()  # calc is asynchronous on `s`
            out["dev"] = f.cpu().numpy()
            assert torch.cuda.current_device() == 0  # restored
        except BaseException as e:  # noqa: BLE001
            out["err"] = e

    t = threading.Thread(target=work)
    t.start()
    t.join()
    assert "err" not in out, out.get("err")
    assert np.array_equal(out["host"], ref) and np.array_equal(out["dev"], ref)
    # a handle belongs to the device of its first call: reuse on another device is refused, not silently run
    alg = ocb.FarnebackOpticalFlow_create(numLevels=3)
    alg.calc_host(I0, I1)                                 # binds to device 0
    with pytest.raises(ocb.B2FError) as e:
        alg.calc(torch.from_numpy(I0).to(d1), torch.from_numpy(I1).to(d1), torch.empty((96, 128, 2), device=d1))
    assert e.value.status == 1


@pytest.mark.parametrize("family,params,dt", [
    ("tvl1", dict(nscales=3, warps=2, epsilon=0.0, iterations=10), "u8"),
    ("farneback", dict(num_levels=3, num_iters=3), "u8"),
    ("brox", dict(inner_iterations=2, outer_iterations=10, solver_iterations=3), "f32")])
def test_native_batch_front_end_equals_per_pair_calc(cuda_device, family, params, dt):
    """b2f_batch_* (csrc/batch.cu): pairs dealt over engine handles on their own streams, forked from and joined
    to the caller's stream -- same bits as one synchronous calc per pair, device and host paths."""
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200.batch import NativeFlowBatch
    frames = _frames(8, 96, 136, dt)
    pairs_h = [(frames[i], frames[i + 1]) for i in range(7)]
    make = {"tvl1": lambda: ocb.OpticalFlowDual_TVL1_create(nscales=3, warps=2, epsilon=0.0, iterations=10),
            "farneback": lambda: ocb.FarnebackOpticalFlow_create(numLevels=3, numIters=3),
            "brox": lambda: ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 3)}[family]
    ref_alg = make()
    want = [ref_alg.calc_host(a, b) for a, b in pairs_h]
    nb = NativeFlowBatch(family, params, n_streams=3)
    # device path on a side stream, bracketed by events on that stream
    s = torch.cuda.Stream(device=cuda_device)
    with torch.cuda.stream(s):
        dev_pairs = [(torch.from_numpy(a).to(cuda_device), torch.from_numpy(b).to(cuda_device)) for a, b in pairs_h]
        flows = torch.zeros((7, 96, 136, 2), device=cuda_device)
        nb.run_device(dev_pairs, [flows[i] for i in range(7)], stream=s)
        done = torch.cuda.Event()
        done.record(s)
    done.synchronize()  # the join made the caller's stream wait for every engine stream
    got = flows.cpu().numpy()
    for i in range(7):
        assert np.array_equal(got[i], want[i]), i
    assert nb.launches() > 0
    # host path: worker threads inside the library
    out = [np.zeros((96, 136, 2), np.float32) for _ in range(7)]
    nb.run_host(pairs_h, out)
    for i in range(7):
        assert np.array_equal(out[i], want[i]), i
    nb.reset_stats()
    assert nb.launches() == 0
    # argument errors propagate as status codes
    with pytest.raises(ocb.B2FError):
        nb.run_host([(frames[0], frames[1][:, :100])], [out[0]])
    nb.close()
