"""The Brox engine against its CUDA-semantics model (oracle/brox_model.c) at the benchmark frame size and at the shapes
where the solver's regions, halos and the prepare kernel's 32 x 8 chunks meet the image edges.

With aux_path 1 the data term's reciprocal square root is correctly rounded and every other operation of the engine is
spelled out in brox.cu, so the flow must equal the model's bit for bit (compared as int32, +0 and -0 equal).  SOR at
omega = 1.99 turns a one-ulp defect into a visible flow change, so nothing looser would see a seam bug.  Every case
first asserts which solver ran on each level and how many iterations each launch fused.

The production path (aux_path 0, rsqrtf) cannot be modelled bit for bit: its error is bounded by 4x the distance
between the exact model and the model with the rsqrt moved by up to 2 ulp (q50, q99, q99.9, max), with small floors.
At full size that bound is weak by nature (rounding alone moves the flow by up to ~1e-2 px); the bit-exact cases carry
the weight."""
import math

import numpy as np
import pytest

from oracle import synth, brox_model as bm, brox_model_native as bn

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not bn.available(), reason="libbrox_model.so not built")]

BENCH = dict(alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=10, outer_iterations=77, solver_iterations=10)
SR = 64


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def expected_paths(h, w, P, kernel_path=0, fused=0, n_sm=132):
    """BroxEngine::solve's dispatch per level (finest first): (b2f_brox_path, iterations of the first launch)."""
    sizes = bm.pyramid_sizes(h, w, P["scale_factor"], P["outer_iterations"])
    out = []
    S = P["solver_iterations"]
    for (lh, lw) in sizes:
        single = lw <= SR and lh <= SR
        it_best = 5
        if not single and fused > 0:
            it_best = fused
        elif not single:
            best = 1e30
            for cand in range(1, min(12, S) + 1):
                t = SR - 4 * cand
                if t < 8:
                    break
                launches = -(-S // cand)
                waves = math.ceil((-(-lw // t)) * (-(-lh // t)) / n_sm)
                cost = launches * (waves * (3.0 + 0.7 * cand) + 2.0)
                if cost < best:
                    best, it_best = cost, cand
        it_best = min(it_best, 13)
        it1 = S if single else min(S, it_best)
        tile = SR if single else SR - 4 * it1
        regions = 1 if single else (-(-lw // tile)) * (-(-lh // tile))
        if kernel_path == 3 and it1 == S and regions <= n_sm:
            out.append((4, it1))
        elif kernel_path == 1:
            out.append((3, 0))
        else:
            out.append((2 if kernel_path == 2 else 1, it1))
    return out


def _run(I0, I1, P, kernel_path=0, aux=1, fused=0, graph=0, stream=False, pitched=False):
    import torch
    import opencv_contrib_b200 as ocb
    dev = torch.device("cuda:0")
    alg = ocb.BroxOpticalFlow_create(**P)
    alg.setEngineOption("kernel_path", kernel_path)
    alg.setEngineOption("aux_path", aux)
    alg.setEngineOption("fused_iters", fused)
    alg.setEngineOption("use_graph", graph)
    h, w = I0.shape
    if pitched:   # ROI views with a row pitch larger than the width, and a pitched flow output
        b0 = torch.zeros((h + 3, w + 7), device=dev)
        b1 = torch.zeros((h + 3, w + 7), device=dev)
        b0[1:h + 1, 2:w + 2] = torch.from_numpy(I0)
        b1[1:h + 1, 2:w + 2] = torch.from_numpy(I1)
        d0, d1 = b0[1:h + 1, 2:w + 2], b1[1:h + 1, 2:w + 2]
        fb = torch.full((h + 2, w + 5, 2), float("nan"), device=dev)
        fout = fb[1:h + 1, 3:w + 3]
        alg.calc(d0, d1, fout)
        torch.cuda.synchronize()
        assert torch.isnan(fb[0]).all() and torch.isnan(fb[:, :3]).all()
        f = fout.cpu().numpy()
    elif stream:
        s = torch.cuda.Stream()
        d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            f = alg.calc(d0, d1, stream=s)
            f2 = alg.calc(d0, d1, stream=s)   # graph replay
        s.synchronize()
        f, f2 = f.cpu().numpy(), f2.cpu().numpy()
        assert _same(f, f2), "graph replay differs"
    else:
        f = alg.calc(torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)).cpu().numpy()
    n = alg.getStats()["levels"]
    return f, [alg.getActivePath(l) for l in range(n)], alg


def _same(a, b):
    return bool(((a.view(np.int32) == b.view(np.int32)) | ((a == 0) & (b == 0))).all())


def _assert_exact(got, ref, what):
    if not _same(got, ref):
        bad = (got != ref).any(axis=-1)
        ys, xs = np.nonzero(bad)
        raise AssertionError(f"{what}: {int(bad.sum())} pixels differ, first at {(int(ys[0]), int(xs[0]))}, "
                             f"max |d| {float(np.abs(got - ref).max()):.3g}, x % 32 of differing: "
                             f"{np.bincount(xs % 32, minlength=32).tolist()}")


def _model(I0, I1, P, rsqrt="exact", counters=None):
    return bn.calc(I0, I1, bm.BroxParams(**P), rsqrt, counters)


def _q(e):
    e = np.abs(e).ravel().astype(np.float64)
    return np.array([np.quantile(e, 0.5), np.quantile(e, 0.99), np.quantile(e, 0.999), e.max()])


def _assert_production(got, exact, pert, floors, what):
    bound = np.maximum(4 * _q(pert - exact), floors)
    err = _q(got - exact)
    print(f"{what}: engine-vs-exact q50/q99/q99.9/max {err}, exact-vs-perturbed {_q(pert - exact)}")
    assert (err <= bound).all(), (what, err.tolist(), bound.tolist())


@pytest.fixture(scope="module")
def bench720():
    I0, I1, _ = synth.make_pair(720, 1280, seed=11, kind="smooth", dtype="f32")
    return I0, I1, _model(I0, I1, BENCH)


@pytest.mark.parametrize("kernel_path", [0, 1, 2, 3])
def test_720p_bench_config_bit_exact(bench720, kernel_path):
    I0, I1, ref = bench720
    got, paths, alg = _run(I0, I1, BENCH, kernel_path=kernel_path, graph=1, stream=True)
    assert paths == expected_paths(720, 1280, BENCH, kernel_path, n_sm=_sms()), paths
    if kernel_path == 0:
        assert paths[0] == (1, 5) and paths[1] == (1, 4), paths[:2]
    if kernel_path == 3:
        assert (4, 10) in paths and paths[0][0] == 1, paths
    _assert_exact(got, ref, f"720p kernel_path {kernel_path}")


def test_720p_production_path(bench720):
    I0, I1, ref = bench720
    got, _, _ = _run(I0, I1, BENCH, aux=0, graph=1, stream=True)
    pert = _model(I0, I1, BENCH, "perturbed")
    _assert_production(got, ref, pert, np.array([1e-4, 2e-3, 5e-3, 2e-2]), "720p production")


def test_1080p_bench_parameters_bit_exact():
    I0, I1, _ = synth.make_pair(1080, 1920, seed=12, kind="smooth", dtype="f32")
    got, paths, _ = _run(I0, I1, BENCH)
    exp = expected_paths(1080, 1920, BENCH, n_sm=_sms())
    assert paths == exp, paths
    tile = SR - 4 * exp[0][1]
    assert -(-1920 // tile) * -(-1080 // tile) > 8 * _sms()   # more than 8 waves of regions on level 0
    _assert_exact(got, _model(I0, I1, BENCH), "1080p")


def _one_level(solver=7, inner=2, **kw):
    return dict(alpha=0.197, gamma=50.0, scale_factor=0.8, inner_iterations=inner, outer_iterations=1,
                solver_iterations=solver, **kw)


def _sweep_shapes(n_sm):
    out = []
    for fused in (2, 3):
        tile = SR - 4 * fused
        for regions in (n_sm, n_sm + 1, 2 * n_sm + 1):
            cols = 12
            rows = -(-regions // cols)
            if rows * cols != regions:       # regions = cols * rows exactly when possible, else the next shape up
                cols = regions
                rows = 1
            out.append((rows * tile - 5, cols * tile - 3, fused))
        for d in (-1, 0, 1):
            out.append((3 * tile + d, 5 * tile + d, fused))
    for d in (63, 64, 65):
        out += [(d, 40, 3), (40, d, 3), (d, d, 3)]
    for wr in (0, 1, 31):
        for hr in (0, 1, 7):
            out.append((8 * 9 + hr, 32 * 5 + wr, 4))
    return out


@pytest.mark.parametrize("case", range(36))
def test_shape_sweep_bit_exact(case):
    shapes = _sweep_shapes(_sms())
    if case >= len(shapes):
        pytest.skip("fewer shapes on this device")
    h, w, fused = shapes[case]
    P = _one_level(solver=7)            # 7 solver iterations: not a multiple of the fused count
    I0, I1, _ = synth.make_pair(h, w, seed=case, kind="smooth", dtype="f32")
    got, paths, _ = _run(I0, I1, P, fused=fused)
    assert paths == expected_paths(h, w, P, fused=fused, n_sm=_sms()), (h, w, paths)
    _assert_exact(got, _model(I0, I1, P), f"{h}x{w} fused {fused}")


def test_cooperative_kernel_at_sm_count_and_fallback():
    n = _sms()
    P = _one_level(solver=10, inner=3)
    tile = SR - 4 * 10                   # all 10 iterations in one launch: 24 x 24 tiles
    for regions, coop in ((n, True), (n + 1, False)):
        cols = next(c for c in range(12, 0, -1) if regions % c == 0) if regions % 12 else 12
        rows = regions // cols
        h, w = rows * tile - 2, cols * tile - 1
        I0, I1, _ = synth.make_pair(h, w, seed=regions, kind="smooth", dtype="f32")
        got, paths, _ = _run(I0, I1, P, kernel_path=3, fused=10)
        assert paths == [((4, 10) if coop else (1, 10))], (regions, paths)
        _assert_exact(got, _model(I0, I1, P), f"coop {regions} regions")


def _special(kind, h, w):
    I0, I1, _ = synth.make_pair(h, w, seed=5, kind="smooth", dtype="f32")
    if kind == "constant":
        return np.full((h, w), 0.25, np.float32), np.full((h, w), 0.75, np.float32)
    if kind == "same":
        return I0, I0.copy()
    if kind == "checker":
        c = ((np.add.outer(np.arange(h), np.arange(w)) & 1)).astype(np.float32)
        return c, 1 - c
    if kind == "x255":
        return I0 * np.float32(255), I1 * np.float32(255)
    if kind == "translation":
        T = synth.make_pair(h + 64, w + 64, seed=6, kind="smooth", dtype="f32")[0]
        return T[:h, :w].copy(), T[40:40 + h, 50:50 + w].copy()
    raise ValueError(kind)


@pytest.mark.parametrize("h,w,P", [
    (1, 37, _one_level(solver=3)), (37, 1, _one_level(solver=3)), (2, 2, _one_level(solver=3)),
    (15, 200, _one_level(solver=5)),
    (90, 120, dict(BENCH, scale_factor=0.5, inner_iterations=3, solver_iterations=4)),
    (70, 90, dict(BENCH, scale_factor=0.95, outer_iterations=12, inner_iterations=2, solver_iterations=3)),
    (96, 128, dict(BENCH, gamma=0.0, inner_iterations=3, solver_iterations=4)),
])
def test_parameter_edges_bit_exact(h, w, P):
    rng = np.random.default_rng(h * w)
    I0, I1 = rng.random((h, w), dtype=np.float32), rng.random((h, w), dtype=np.float32)
    got, paths, _ = _run(I0, I1, P)
    assert paths == expected_paths(h, w, P, n_sm=_sms()), paths
    c = {}
    ref = _model(I0, I1, P, counters=c)
    assert c["levels"] == len(paths)
    _assert_exact(got, ref, f"{h}x{w} {P}")
    if P["outer_iterations"] == 1:   # the production path on one level: rounding barely grows, so the bound is tight
        prod, _, _ = _run(I0, I1, P, aux=0)
        _assert_production(prod, ref, _model(I0, I1, P, "perturbed"), np.array([1e-7, 1e-6, 2e-6, 1e-5]),
                           f"{h}x{w} production")


@pytest.mark.parametrize("kind", ["constant", "same", "checker", "x255", "translation"])
def test_special_inputs_bit_exact(kind):
    h, w = 100, 140
    P = dict(BENCH, inner_iterations=3, solver_iterations=4)
    I0, I1 = _special(kind, h, w)
    got, paths, _ = _run(I0, I1, P)
    assert paths == expected_paths(h, w, P, n_sm=_sms())
    c = {}
    ref = _model(I0, I1, P, counters=c)
    assert np.isfinite(ref).all()
    if kind == "translation":
        # the image borders alone account for at most 2 (h + w) fetches per level, < 2 (h + w) / (1 - 0.8) in all: more
        # means interior pixels were warped out of the image
        assert c["mirrored"] > h * w // 4 > 2 * (h + w) * 5, c
    _assert_exact(got, ref, kind)


def test_pitched_inputs_and_output_bit_exact():
    h, w = 131, 170
    P = dict(BENCH, inner_iterations=3, solver_iterations=5)
    I0, I1, _ = synth.make_pair(h, w, seed=8, kind="smooth", dtype="f32")
    got, _, _ = _run(I0, I1, P, pitched=True, graph=1)
    _assert_exact(got, _model(I0, I1, P), "pitched")


def test_active_path_rejects_unsolved_level():
    import opencv_contrib_b200 as ocb
    I0, I1, _ = synth.make_pair(40, 50, seed=1, kind="smooth", dtype="f32")
    _, paths, alg = _run(I0, I1, _one_level(solver=2))
    assert len(paths) == 1
    with pytest.raises(ocb.B2FError):
        alg.getActivePath(1)
