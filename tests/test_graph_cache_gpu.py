"""GPU tests of the host-side lifecycle every graph engine shares: a calc on a real stream captures the fixed schedule
in a CUDA graph once per key and replays it afterwards.  The graph must change nothing a caller can see: the flow,
the launch and byte accounting of getStats(), the iteration count and the per-level active paths equal those of the
eager schedule; a handle whose parameters, knobs or frame size changed and changed back equals a fresh handle; and
fresh handles driven concurrently by the native batch's host threads equal per-pair calls."""
import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu

SHAPE, OTHER_SHAPE = (96, 136), (80, 120)


def _make(name):
    import opencv_contrib_b200 as ocb
    return {
        "tvl1": lambda: ocb.OpticalFlowDual_TVL1_create(nscales=3, warps=2, epsilon=0.0, iterations=10),
        "tvl1_eps": lambda: ocb.OpticalFlowDual_TVL1_create(nscales=3, warps=2, epsilon=0.01, iterations=40),
        "farneback": lambda: ocb.FarnebackOpticalFlow_create(numLevels=3, numIters=3),
        "brox": lambda: ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 3),
        "deepflow": lambda: ocb.createOptFlow_DeepFlow(fixedPointIterations=2, sorIterations=6),
        "dis": lambda: ocb.DISOpticalFlow_create(ocb.DISOPTICAL_FLOW_PRESET_FAST),
    }[name]()


# (setter, value) pairs: a parameter the schedule depends on, and a knob the engine reads (None: it reads none)
PARAM_CHANGE = {"tvl1": ("setNumWarps", 3), "tvl1_eps": ("setEpsilon", 0.05), "farneback": ("setNumIters", 4),
                "brox": ("setInnerIterations", 3), "deepflow": ("setSorIterations", 8), "dis": ("setFinestScale", 1)}
# TV-L1 with epsilon > 0 and kernel_path 1 runs without a graph: changing back must find the graph captured before
KNOB_CHANGE = {"tvl1": ("fused_iters", 4), "tvl1_eps": ("kernel_path", 1), "farneback": ("kernel_path", 2),
               "brox": ("fused_iters", 2), "deepflow": None, "dis": None}
BATCH_PARAMS = {"tvl1": ("tvl1", dict(nscales=3, warps=2, epsilon=0.0, iterations=10)),
                "tvl1_eps": ("tvl1", dict(nscales=3, warps=2, epsilon=0.01, iterations=40)),
                "farneback": ("farneback", dict(num_levels=3, num_iters=3)),
                "brox": ("brox", dict(inner_iterations=2, outer_iterations=10, solver_iterations=3)),
                "deepflow": ("deepflow", dict(fixed_point_iterations=2, sor_iterations=6)),
                "dis": ("dis", dict())}
ENGINES = list(PARAM_CHANGE)


def _pair(name, shape, seed=0):
    I0, I1, _ = synth.make_pair(*shape, seed=seed, kind="smooth")
    if name == "brox":
        return I0.astype(np.float32) / 255.0, I1.astype(np.float32) / 255.0
    return I0, I1


def _paths(alg):
    """Every level's active path; DIS numbers them by pyramid scale, starting at its finest scale."""
    first = alg.getFinestScale() if hasattr(alg, "getFinestScale") else 0
    levels = alg.getStats()["levels"]
    from opencv_contrib_b200._lib import PARAM
    return [alg._get(PARAM["engine"]["active_path"] + first + i) for i in range(levels)]


def _accounting(alg):
    s = alg.getStats()
    return s["launches"], s["iterations_run"], {k: (v["launches"], v["bytes"]) for k, v in s["classes"].items()}


def _calc(alg, pair, stream):
    import torch
    dev = stream.device
    f = alg.calc(torch.from_numpy(pair[0]).to(dev), torch.from_numpy(pair[1]).to(dev), stream=stream)
    stream.synchronize()
    return f.cpu().numpy()


@pytest.mark.parametrize("name", ENGINES)
def test_graph_equals_eager_schedule(cuda_device, name):
    """use_graph 1 against 0 on a real stream, call by call: the capturing call and the replaying call.  TV-L1 with
    epsilon > 0 decides its stopping rule on the host without a graph and launches differently, so only its flow and
    iteration count are compared."""
    import torch
    s = torch.cuda.Stream(device=cuda_device)
    graph, eager = _make(name), _make(name)
    graph.setEngineOption("use_graph", 1)
    eager.setEngineOption("use_graph", 0)
    pairs = [_pair(name, SHAPE, 0), _pair(name, SHAPE, 0), _pair(name, SHAPE, 1)]
    flows = []
    for i, p in enumerate(pairs):
        g, e = _calc(graph, p, s), _calc(eager, p, s)
        assert np.array_equal(g.view(np.uint32), e.view(np.uint32)), (i, float(np.abs(g - e).max()))
        flows.append(g)
        (gl, gi, gc), (el, ei, ec) = _accounting(graph), _accounting(eager)
        assert gi == ei > 0, i
        if name != "tvl1_eps":
            assert gl == el, i
            # cumulative byte counts are sums of integers well below 2**53: exact in double
            assert gc == ec, i
            assert _paths(graph) == _paths(eager), i
    assert np.array_equal(flows[0], flows[1])  # replay equals capture


@pytest.mark.parametrize("name", ENGINES)
def test_key_changes_match_fresh_handle(cuda_device, name):
    """On one handle: change a parameter, a knob the engine reads and the frame size in turn, each time changing it
    back.  Every result and its active paths equal those of a fresh handle configured the same way."""
    import torch
    s = torch.cuda.Stream(device=cuda_device)
    setter, value = PARAM_CHANGE[name]
    knob = KNOB_CHANGE[name]
    steps = [dict()]
    steps += [dict(param=value), dict()]
    if knob:
        steps += [dict(knob=knob[1]), dict()]
    steps += [dict(shape=OTHER_SHAPE), dict()]

    default = getattr(_make(name), "get" + setter[3:])()

    def configure(alg, step):
        getattr(alg, setter)(step.get("param", default))
        if knob:
            alg.setEngineOption(knob[0], step.get("knob", 0))

    live = _make(name)
    for i, step in enumerate(steps):
        configure(live, step)
        pair = _pair(name, step.get("shape", SHAPE), seed=i)
        got = _calc(live, pair, s)
        fresh = _make(name)
        configure(fresh, step)
        want = _calc(fresh, pair, s)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (i, step)
        assert _paths(live) == _paths(fresh), (i, step)
        assert live.getStats()["iterations_run"] == fresh.getStats()["iterations_run"], (i, step)


@pytest.mark.parametrize("name", ENGINES)
def test_native_batch_host_threads_equal_per_pair_calc(cuda_device, name):
    """Fresh engines on 4 streams, each driven by its own host thread (their first calls, which capture, run
    concurrently), equal one calc per pair."""
    from opencv_contrib_b200.batch import NativeFlowBatch
    family, params = BATCH_PARAMS[name]
    pairs = [_pair(name, SHAPE, seed=i) for i in range(8)]
    ref = _make(name)
    want = [ref.calc_host(a, b) for a, b in pairs]
    nb = NativeFlowBatch(family, params, n_streams=4)
    out = [np.zeros(SHAPE + (2,), np.float32) for _ in pairs]
    nb.run_host(pairs, out)
    for i in range(len(pairs)):
        assert np.array_equal(out[i].view(np.uint32), want[i].view(np.uint32)), i
    nb.close()
