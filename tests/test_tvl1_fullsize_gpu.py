"""TV-L1 engine vs the native CUDA-semantics model (oracle/tvl1_gpu_model.c) at the sizes and shapes the production
dispatch actually sees: persistent CTAs that take a second region and a wave tail, TMA box origins at every column
residue, the tiled warp kernel's switch to the separable fallback, sub-region images, and the BASELINE frame sizes.

Default knobs, CUDA graph on, a real stream.  Every case first asserts which kernels ran (getActivePath), so a
shape that silently falls back to the plain-load kernels fails instead of passing vacuously.

The engine is compared with the engine-rounding model ("eng" build, fed this device's rcp.approx / sqrt.approx
tables) bit for bit, as uint32 views, in every case: the shape sweep, both BASELINE sizes on the TMA and the unfused
kernels, the staged-window fallback at every initial-flow amplitude, and the reference defaults whenever the engine ran
as many iterations as the model.  The tolerances that used to bound the engine now bound that model against the float
model, with the double model as the yardstick (see DESIGN.md "Parity"), so the engine inherits them:
  * staged-window fallback (1080p, one level, initial flows up to 40 px): max |dflow| <= 1e-3 px;
  * shape sweep (one level, 2 warps x 30 iterations = passes of 8 + 8 + 8 + 6): max |dflow| <= 1e-3 px and the 99 %
    quantile <= 1e-4 px, each raised to 4 x the float-vs-double figure where float rounding alone moves the flow
    further (2513 x 221, seed 22: one ill-conditioned pixel moves 5.1e-3 px between the float and the double model);
  * BASELINE sizes (5 scales x 10 warps x 30 iterations): at the 50 %, 99 %, 99.9 % quantiles and the max, at most
    4 x the float model's distance from the double model on the same input (at 1080p the max of that is ~0.02 px);
  * reference defaults at 1080p (epsilon = 0.01, device-side WHILE loop): the iteration count equals the model's
    per-warp trace summed, unless a sampled error sum lay within 1e-5 (relative) of its threshold (the device sums
    its error image in another order than the model); the flow as in the sweep.
"""
import time

import numpy as np
import pytest

from oracle import metrics, mufu, synth, tvl1_gpu_model as gm, tvl1_gpu_model_native as nm

pytestmark = pytest.mark.gpu

TILE = 48      # centre tile of a 64 x 64 region at the 8-pixel halo of the 8- and 6-iteration passes
WB_W, WB_H = 88, 56  # the tiled warp kernel's staged box; smaller levels take the separable kernel
SWEEP = dict(nscales=1, warps=2, epsilon=0.0, iterations=30)
BASELINE = dict(nscales=5, warps=10, epsilon=0.0, iterations=30)
FACTOR = 4.0
QUANTILES = (0.5, 0.99, 0.999, 1.0)
FLOORS = {0.99: 1e-4, 1.0: 1e-3}  # the small-size bounds, for the sweep and the epsilon run


def _check_vs_yardstick(e, yard, floors, label):
    """Quantiles of e = EPE(engine-rounding model, float model) against FACTOR x the same quantiles of
    yard = EPE(float model, double model); floors: {quantile: bound} checked instead wherever it is the larger (None:
    all QUANTILES, no floor)."""
    for q in (QUANTILES if floors is None else sorted(floors)):
        v, y = float(np.quantile(e, q)), float(np.quantile(yard, q))
        bound = max(FACTOR * y, 0.0 if floors is None else floors[q])
        print(f"{label}: q{q:g} eng-vs-f32 {v:.2e}, f32-vs-f64 {y:.2e}, bound {bound:.2e}")
        assert v <= bound, (label, q, v, y, _worst_tiles(e))


def _assert_bits(got, exact, label):
    """The engine equals the engine-rounding model bit for bit; on failure, how many values differ and the worst
    pixels with their position in the 48 x 48 centre tile."""
    assert got.shape == exact.shape and exact.dtype == np.float32, (label, got.shape, exact.shape)
    diff = got.view(np.uint32) != exact.view(np.uint32)
    assert not diff.any(), (label, int(diff.sum()), _worst_tiles(metrics.epe(got, exact)))


@pytest.fixture(scope="module", autouse=True)
def _native_model(cuda_device):
    if not (nm.available("f32") and nm.available("f64") and nm.available("eng")):
        pytest.fail("oracle/_build/libtvl1_gpu_model_{f32,f64,eng}.so missing: run build()")
    nm.set_mufu_tables(*mufu.device_tables(cuda_device))


@pytest.fixture(scope="module")
def stream(cuda_device):
    import torch
    return torch.cuda.Stream(device=cuda_device)


@pytest.fixture(scope="module")
def num_sms(cuda_device):
    import torch
    return torch.cuda.get_device_properties(cuda_device).multi_processor_count


def _engine(dev, stream, I0, I1, path=0, init=None, **kw):
    import torch
    import opencv_contrib_b200 as ocb
    alg = ocb.OpticalFlowDual_TVL1_create(**kw)
    alg.setEngineOption("kernel_path", path)
    assert alg.getEngineOption("use_graph") == 1 and alg.getEngineOption("aux_path") == 0
    d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
    fl = None if init is None else torch.from_numpy(np.ascontiguousarray(init)).to(dev)
    f = alg.calc(d0, d1, fl, stream)
    stream.synchronize()
    return f.cpu().numpy(), alg


def _expected_paths(h, w, P, iter_flags):
    from opencv_contrib_b200._lib import TVL1_PATH
    sizes, ns = gm.level_sizes(h, w, P.nscales, P.scaleStep)
    return [iter_flags | (TVL1_PATH["warp_tiled"] if (c >= WB_W and r >= WB_H) else TVL1_PATH["warp_untiled"])
            for r, c in sizes[:ns]]


def _check_paths(alg, h, w, P, iter_flags):
    want = _expected_paths(h, w, P, iter_flags)
    got = [alg.getActivePath(s) for s in range(len(want))]
    assert got == want, f"{h}x{w}: kernels that ran per level {got}, expected {want}"
    return got


def _pair(h, w, seed, dtype):
    """A synthetic pair cropped to h x w (synth needs a few pixels of texture)."""
    I0, I1, _ = synth.make_pair(max(h, 16), max(w, 16), seed=seed, kind="smooth", dtype=dtype)
    return np.ascontiguousarray(I0[:h, :w]), np.ascontiguousarray(I1[:h, :w])


def _worst_tiles(e, n=8):
    """Coordinates of the n worst pixels inside their 48 x 48 centre tile: a seam defect shows as x or y mod 48 in
    {0, 47} at every one of them."""
    idx = np.argsort(e, axis=None)[-n:][::-1]
    ys, xs = np.unravel_index(idx, e.shape)
    return [dict(x=int(x), y=int(y), x_mod48=int(x % TILE), y_mod48=int(y % TILE), epe=float(e[y, x]))
            for y, x in zip(ys, xs)]


def _sweep_shapes(n_sm):
    """(rows, cols, why): region counts from the device's SM count, column residues mod 4 at two or more waves,
    the tiled warp kernel's 88 x 56 threshold, and images smaller than one region."""
    def grid(n, rx=29, ry=17):  # tx * ty == n regions, ragged right and bottom edges
        tx = max(d for d in range(1, int(n ** 0.5) + 1) if n % d == 0)
        ty = n // tx
        return (ty - 1) * TILE + ry, (tx - 1) * TILE + rx
    shapes = [(*grid(n), f"{n} regions") for n in (n_sm, n_sm + 1, 2 * n_sm + 1)]
    ty = 12
    tx = -(-(2 * n_sm + 1) // ty)  # at least 2 n_SM + 1 regions
    shapes += [((ty - 1) * TILE + 12, (tx - 1) * TILE + r, f"cols % 4 == {((tx - 1) * TILE + r) % 4}, {tx * ty} regions")
               for r in (29, 30, 31, 32)]
    shapes += [(57, c, "warp box threshold") for c in (87, 88, 89)] + [(r, 89, "warp box threshold") for r in (55, 56)]
    shapes += [(1, 37, "1xN"), (37, 1, "Nx1"), (2, 2, "2x2"), (40, 45, "below one region")]
    return shapes


def test_shape_sweep_vs_native_model(cuda_device, stream, num_sms):
    from opencv_contrib_b200._lib import TVL1_PATH
    P = gm.TVL1Params(**SWEEP)
    t0 = time.time()
    for i, (h, w, why) in enumerate(_sweep_shapes(num_sms)):
        dtype = "f32" if i % 2 else "u8"
        I0, I1 = _pair(h, w, seed=20 + i, dtype=dtype)
        got, alg = _engine(cuda_device, stream, I0, I1, **SWEEP)
        paths = _check_paths(alg, h, w, P, TVL1_PATH["iter_tma"])
        exact = nm.calc(I0, I1, P, precision="eng")
        ref = nm.calc(I0, I1, P)
        yard = metrics.epe(ref, nm.calc(I0, I1, P, precision="f64"))
        print(f"sweep {h}x{w} {dtype} ({why}): regions {-(-w // TILE) * -(-h // TILE)} on {num_sms} SMs, "
              f"active path {paths}")
        assert np.isfinite(got).all()
        _assert_bits(got, exact, f"{h}x{w}")
        _check_vs_yardstick(metrics.epe(exact, ref), yard, FLOORS, f"  {h}x{w}")
    print(f"sweep: {time.time() - t0:.1f} s")


@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
def test_baseline_size_vs_native_model(cuda_device, stream, h, w):
    from opencv_contrib_b200._lib import TVL1_PATH
    I0, I1, _ = synth.make_pair(h, w, seed=0, kind="smooth")
    P = gm.TVL1Params(**BASELINE)
    t0 = time.time()
    exact = nm.calc(I0, I1, P, precision="eng")
    t_eng = time.time() - t0
    ref = nm.calc(I0, I1, P)
    yard = metrics.epe(ref, nm.calc(I0, I1, P, precision="f64"))
    t_model = time.time() - t0 - t_eng
    _check_vs_yardstick(metrics.epe(exact, ref), yard, None, f"{w}x{h} model")
    for path, flags in ((0, TVL1_PATH["iter_tma"]), (1, TVL1_PATH["iter_unfused"])):
        got, alg = _engine(cuda_device, stream, I0, I1, path=path, **BASELINE)
        paths = _check_paths(alg, h, w, P, flags)
        assert np.isfinite(got).all()
        _assert_bits(got, exact, f"{w}x{h} path {path} {paths}")
    print(f"{w}x{h}: engine-rounding model {t_eng:.1f} s, float + double model {t_model:.1f} s")


def test_staged_window_fallback_multi_wave(cuda_device, stream):
    """One 1080p level (920 regions, several waves), initial flows from sub-pixel to far beyond the warp kernel's
    12-pixel staged margin, part of them pointing out of the image."""
    from opencv_contrib_b200._lib import TVL1_PATH
    h, w = 1080, 1920
    I0, I1, _ = synth.make_pair(h, w, seed=3, kind="smooth")
    P = gm.TVL1Params(nscales=1, warps=2, epsilon=0.0, iterations=10, useInitialFlow=True)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    rng = np.random.default_rng(7)
    for amp in (0.7, 6.0, 11.5, 40.0):
        init = np.stack([amp * np.sin(xx / 37.0 + yy / 53.0), amp * np.cos(xx / 41.0 - yy / 29.0)], axis=-1)
        init = (init + rng.uniform(-0.5, 0.5, init.shape)).astype(np.float32)
        got, alg = _engine(cuda_device, stream, I0, I1, init=init, nscales=1, warps=2, epsilon=0.0, iterations=10,
                           useInitialFlow=True)
        paths = _check_paths(alg, h, w, P, TVL1_PATH["iter_tma"])
        exact = nm.calc(I0, I1, P, init_flow=init, precision="eng")
        e = metrics.epe(exact, nm.calc(I0, I1, P, init_flow=init))
        print(f"staged window amp {amp}: active path {paths}, model eng-vs-f32 max |dflow| {e.max():.2e}")
        assert np.isfinite(got).all()
        _assert_bits(got, exact, f"staged window amp {amp}")
        assert e.max() <= 1e-3, (amp, _worst_tiles(e))


def test_reference_defaults_iteration_trace_1080p(cuda_device, stream):
    """create() defaults (5 scales, 5 warps, epsilon 0.01, up to 300 iterations): the reference's stopping rule runs on
    the GPU as a WHILE conditional node.  The engine reports the total number of inner iterations; it must equal the
    engine-rounding model's per-warp counts summed, and then the flow is bit for bit the model's.  A difference is only
    excusable where a sampled error sum lay within 1e-5 (relative) of scaledEpsilon: the device sums its error image
    in another order than the model, so there it may decide the other way."""
    from opencv_contrib_b200._lib import TVL1_PATH
    h, w = 1080, 1920
    I0, I1, _ = synth.make_pair(h, w, seed=5, kind="smooth")
    P = gm.TVL1Params()
    trace, ratios = [], []
    exact = nm.calc(I0, I1, P, trace=trace, ratios=ratios, precision="eng")
    ref = nm.calc(I0, I1, P)
    yard = metrics.epe(ref, nm.calc(I0, I1, P, precision="f64"))
    got, alg = _engine(cuda_device, stream, I0, I1)
    paths = _check_paths(alg, h, w, P, TVL1_PATH["iter_tma"] | TVL1_PATH["iter_unfused"])
    closest = min(abs(r - 1.0) for r in ratios)
    n_engine, n_model = alg.getStats()["iterations_run"], sum(sum(t) for t in trace)
    print(f"defaults 1080p: active path {paths}; iterations engine {n_engine}, model {n_model} (per level and warp "
          f"{trace}); closest sampled error sum {closest:.2e} from its threshold")
    assert np.isfinite(got).all()
    if n_engine != n_model:
        assert closest <= 1e-5, (n_engine, n_model, trace, closest)
    else:
        _assert_bits(got, exact, "defaults 1080p")
        _check_vs_yardstick(metrics.epe(exact, ref), yard, FLOORS, "defaults 1080p")
