"""interpolateFrames (csrc/frames.cu) against oracle/interpolate_model.py.

(a) Order-free inputs: flows on a coarse dyadic grid and a dyadic ``pos`` put every contribution to every
    accumulator on a 2^-k lattice with magnitudes summing below 2^(24-k), so every order of the float atomics
    gives the same bits.  Each case asserts that condition from the model first, then requires the output
    and all six scratch planes bit for bit, at every pixel.
(b) Generic inputs: the blend is a deterministic function of what the call leaves in ``buf``, so the model's
    blend stage fed with the GPU's own ``buf`` must give the output bit for bit; the scratch planes must lie
    within the rounding bound of float summation in any order, carried through the normalisation.

Every call gets a ``buf`` and an output filled with garbage, as views of wider allocations: the call must
clear the view and leave the columns past the view alone.
"""
import numpy as np
import pytest

from oracle import synth, interpolate_model as im

pytestmark = pytest.mark.gpu


def _dyadic(rng, shape, step, lim):
    """Multiples of ``step`` in [-lim, lim]."""
    n = int(round(lim / step))
    return (rng.integers(-n, n + 1, shape) * step).astype(np.float32)


def _smooth_dyadic(h, w, seed, step=0.125, mag=6.0):
    fl = synth.flow_field(h, w, "smooth", seed=seed, mag=mag)
    return (np.round(fl / step) * step).astype(np.float32)


def _frames(rng, h, w):
    return rng.random((h, w), dtype=np.float32), rng.normal(0.5, 0.3, (h, w)).astype(np.float32)


def _garbage(rng, shape):
    g = rng.normal(0, 1e3, shape).astype(np.float32)
    g.flat[::7] = np.nan
    return g


def _run(dev, planes, pos, corrected, pitch, side_stream=False, seed=0):
    """One call on pitched views; returns (out (h, w), buf (6, h, w)).  Asserts that the columns past the views
    still hold what they held before the call."""
    import torch
    import opencv_contrib_b200 as ocb
    h, w = planes[0].shape
    rng = np.random.default_rng(seed)

    def pitched(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        return t, t[:, :w]

    ins = []
    for a in planes:
        full = np.zeros((h, pitch), np.float32)
        full[:, :w] = a
        ins.append(pitched(full)[1])
    out_host, buf_host = _garbage(rng, (h, pitch)), _garbage(rng, (6 * h, pitch))
    out_full, out = pitched(out_host)
    buf_full, buf = pitched(buf_host)
    if side_stream:
        ready = torch.cuda.Event()
        ready.record()  # inputs were written on the current stream
        s = torch.cuda.Stream(device=dev)
        s.wait_event(ready)
        with torch.cuda.stream(s):
            ocb.interpolateFrames(*ins, pos, out, buf, stream=s, corrected=corrected)
            done = torch.cuda.Event()
            done.record(s)
        torch.cuda.current_stream().wait_event(done)
    else:
        ocb.interpolateFrames(*ins, pos, out, buf, corrected=corrected)
    got_out, got_buf = out_full.cpu().numpy(), buf_full.cpu().numpy()
    u32 = lambda a: a.view(np.uint32)
    assert np.array_equal(u32(got_out[:, w:]), u32(out_host[:, w:])), "output padding written"
    assert np.array_equal(u32(got_buf[:, w:]), u32(buf_host[:, w:])), "buf padding written"
    return got_out[:, :w], got_buf.reshape(6, h, pitch)[:, :, :w]


def _engine_model(planes, pos, corrected, pitch):
    """The model's stages in the engine's order; asserts first that every accumulator is order-free."""
    h, w = planes[0].shape
    con = im.splat(*planes[2:], pos, w, h, pitch)
    for p in im.PLANES:
        free = im.order_free(im.terms(con[p], h * pitch))
        assert free.all(), (p, int((~free).sum()))
    acc = [im.accumulate(con[p], h * pitch) for p in im.PLANES]
    buf = im.normalise(acc, corrected, w, h, pitch).reshape(6, h, pitch)[:, :, :w]
    return im.blend(planes[0], planes[1], buf, pos, corrected), buf, con


def _assert_bits(got, want, what):
    g, m = got.view(np.uint32), want.view(np.uint32)
    bad = g != m
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())


def _exact(dev, planes, pos, corrected, pitch, **kw):
    want, wbuf, con = _engine_model(planes, pos, corrected, pitch)
    got, gbuf = _run(dev, planes, pos, corrected, pitch, **kw)
    for k, name in enumerate(im.PLANES):
        _assert_bits(gbuf[k], wbuf[k], name)
    _assert_bits(got, want, "output")
    return wbuf, con


# --------------------------------------------------------------------------------------- (a) bit for bit
@pytest.mark.parametrize("corrected", [False, True])
@pytest.mark.parametrize("pitch", [1920, 2048])
def test_exact_1080p(cuda_device, corrected, pitch):
    """The benchmark's frame size; with a 2048-float pitch the reference mode's coverage clear (by width)
    leaves rows 1013.. accumulated twice."""
    h, w = 1080, 1920
    rng = np.random.default_rng(pitch)
    f0, f1 = _frames(rng, h, w)
    fl = _smooth_dyadic(h, w, 5)
    bl = (-fl + _dyadic(rng, (h, w, 2), 0.125, 0.5)).astype(np.float32)
    wbuf, _ = _exact(cuda_device, [f0, f1, fl[..., 0], fl[..., 1], bl[..., 0], bl[..., 1]], 0.5, corrected, pitch)
    if not corrected and pitch > w:
        jj, ii = np.meshgrid(np.arange(w), np.arange(h))
        assert (ii * pitch + jj >= w * h).mean() > 0.05  # the doubled region is part of the comparison


@pytest.mark.parametrize("corrected", [False, True])
@pytest.mark.parametrize("h,w", [(1, 1), (1, 37), (37, 1), (9, 33), (75, 101), (64, 96)])
def test_exact_grid_tails(cuda_device, corrected, h, w):
    """Partial 32x8 splat blocks and 32x4 blend blocks, pitch 128 (64x96 contiguous)."""
    pitch = w if (h, w) == (64, 96) else 128
    rng = np.random.default_rng(h * 1000 + w)
    f0, f1 = _frames(rng, h, w)
    fl = _dyadic(rng, (h, w, 2), 0.125, 3.0)
    bl = (-fl + _dyadic(rng, (h, w, 2), 0.125, 0.25)).astype(np.float32)
    for pos in (0.25, 0.5):
        _exact(cuda_device, [f0, f1, fl[..., 0], fl[..., 1], bl[..., 0], bl[..., 1]], pos, corrected, pitch,
               seed=int(pos * 4))


@pytest.mark.parametrize("corrected", [False, True])
def test_exact_flows_leave_every_side_and_hit_the_sampling_clamp(cuda_device, corrected):
    """Backward flows pointing out of the frame on all four sides, forward flows of up to 40 px either way on a
    40x56 frame: splat taps fall outside, and the blend's sample coordinates pass the [-2, size + 1] clamp."""
    h, w, pitch = 40, 56, 64
    rng = np.random.default_rng(7)
    f0, f1 = _frames(rng, h, w)
    jj, ii = np.meshgrid(np.arange(w), np.arange(h))
    fu, fv = _dyadic(rng, (h, w), 0.25, 40), _dyadic(rng, (h, w), 0.25, 40)
    bu = (np.round((jj - (w - 1) / 2) * 4) / 4 + _dyadic(rng, (h, w), 0.25, 1)).astype(np.float32)
    bv = (np.round((ii - (h - 1) / 2) * 4) / 4 + _dyadic(rng, (h, w), 0.25, 1)).astype(np.float32)
    for pos in (0.25, 0.75):
        wbuf, _ = _exact(cuda_device, [f0, f1, fu, fv, bu, bv], pos, corrected, pitch)
        # sources whose taps all miss the frame, through each side, in both splats
        for u, v, t in ((fu, fv, pos), (bu, bv, 1 - pos)):
            cx, cy = u * np.float32(t) + jj + 1, v * np.float32(t) + ii + 1
            for side in (cx < 0, cx > w + 1, cy < 0, cy > h + 1):
                assert side.sum() >= 10
        # second samples of the both-visible branch (x + u (1 - pos), less 0.5) below -2 or above size + 1
        both = im.blend_branches(wbuf[0], wbuf[1])[0]
        sx, sy = jj + wbuf[2] * np.float32(1 - pos), ii + wbuf[3] * np.float32(1 - pos)
        for side in (sx < -3, sx > w + 2, sy < -3, sy > h + 2):
            assert (side & both).sum() >= 10


@pytest.mark.parametrize("corrected", [False, True])
def test_exact_negative_weight_taps_at_left_and_top_edges(cuda_device, corrected):
    """u * t in (-2, -1) puts cx in (-1, 0) at column 0: modff gives a negative fraction, so the taps kept in
    column 0 carry negative weights (rows alike).  pos = 0.25: t = 0.25 forward, 0.75 backward."""
    h, w, pitch = 24, 40, 48
    rng = np.random.default_rng(11)
    f0, f1 = _frames(rng, h, w)
    fu, fv = ((-6 + _dyadic(rng, (h, w), 0.125, 1.875)).astype(np.float32) for _ in range(2))  # u/4 in (-2, -1)
    bu, bv = ((-2 + _dyadic(rng, (h, w), 0.125, 0.625)).astype(np.float32) for _ in range(2))  # 3u/4 in (-2, -1)
    _, con = _exact(cuda_device, [f0, f1, fu, fv, bu, bv], 0.25, corrected, pitch)
    assert (con["cov0"].val < 0).sum() >= 100 and (con["cov1"].val < 0).sum() >= 100


@pytest.mark.parametrize("corrected", [False, True])
@pytest.mark.parametrize("pos", [0.0, 1.0])
def test_exact_pos_at_the_ends(cuda_device, corrected, pos):
    h, w, pitch = 48, 70, 80
    rng = np.random.default_rng(13)
    f0, f1 = _frames(rng, h, w)
    fl = _smooth_dyadic(h, w, 2, mag=5.0)
    bl = (-fl + _dyadic(rng, (h, w, 2), 0.125, 0.5)).astype(np.float32)
    _exact(cuda_device, [f0, f1, fl[..., 0], fl[..., 1], bl[..., 0], bl[..., 1]], pos, corrected, pitch)


def _holes(h, w, seed):
    """Piecewise-constant flows on 12x12 blocks: gaps and overlaps at block edges, forward and backward
    independent, so every blend branch takes a visible share of the pixels."""
    rng = np.random.default_rng(seed)
    f0, f1 = _frames(rng, h, w)
    blocks = lambda: np.kron(_dyadic(rng, (h // 12 + 1, w // 12 + 1), 0.5, 6), np.ones((12, 12)))[:h, :w]
    return [f0, f1] + [blocks().astype(np.float32) for _ in range(4)]


@pytest.mark.parametrize("corrected", [False, True])
def test_exact_every_blend_branch(cuda_device, corrected):
    h, w, pitch = 96, 132, 160
    planes = _holes(h, w, 17)
    for pos in (0.25, 0.5, 0.75):
        wbuf, _ = _exact(cuda_device, planes, pos, corrected, pitch)
        shares = [float(m.mean()) for m in im.blend_branches(wbuf[0], wbuf[1])]
        print("pos", pos, "branch shares (both, first only, second only):", shares)
        assert shares[0] > 0.5 and shares[1] > 0.015 and shares[2] > 0.015, shares


@pytest.mark.parametrize("corrected", [False, True])
def test_exact_on_a_side_stream(cuda_device, corrected):
    """The call ordered on a side stream by events, its inputs written on the current stream."""
    h, w = 75, 101
    rng = np.random.default_rng(19)
    f0, f1 = _frames(rng, h, w)
    fl = _smooth_dyadic(h, w, 3)
    bl = (-fl + _dyadic(rng, (h, w, 2), 0.125, 0.25)).astype(np.float32)
    _exact(cuda_device, [f0, f1, fl[..., 0], fl[..., 1], bl[..., 0], bl[..., 1]], 0.25, corrected, 128,
           side_stream=True)


# ------------------------------------------------------------------ (b) generic inputs: exact blend, bounds
def _generic(kind, h, w):
    rng = np.random.default_rng(h + w)
    if kind == "bench":  # bench.py's inputs: per-pixel N(0, 3) flows, bu = -u
        f0, f1 = _frames(rng, h, w)
        u, v = (rng.normal(0, 3, (h, w)).astype(np.float32) for _ in range(2))
        return [f0, f1, u, v, -u, -v]
    if kind == "holes":  # the piecewise-constant flows of (a), off the dyadic grid
        planes = _holes(h, w, 23)
        return planes[:2] + [(p + rng.normal(0, 0.3, (h, w))).astype(np.float32) for p in planes[2:]]
    f0 = (synth.texture(h, w, 1) / 255).astype(np.float32)
    f1 = (synth.texture(h, w, 2) / 255).astype(np.float32)
    fl = synth.flow_field(h, w, "smooth", seed=3)
    bl = -fl + rng.normal(0, 0.05, (h, w, 2)).astype(np.float32)
    return [f0, f1, fl[..., 0], fl[..., 1], bl[..., 0], bl[..., 1]]


@pytest.mark.parametrize("corrected", [False, True])
@pytest.mark.parametrize("kind,h,w,pitch", [("smooth", 64, 96, 96), ("smooth", 75, 101, 128), ("holes", 96, 132, 160),
                                            ("smooth", 1080, 1920, 1920), ("bench", 1080, 1920, 1920)])
def test_generic_blend_exact_and_accumulators_bounded(cuda_device, corrected, kind, h, w, pitch):
    planes = _generic(kind, h, w)
    seen = np.zeros(3, np.int64)
    for pos in (0.5, 0.2):
        got, gbuf = _run(cuda_device, planes, pos, corrected, pitch)
        assert np.isfinite(gbuf).all() and np.isfinite(got).all()
        # the blend: exact at every pixel, from the GPU's own scratch planes
        _assert_bits(got, im.blend(planes[0], planes[1], gbuf, pos, corrected), "output from the GPU's buf")
        shares = [int(m.sum()) for m in im.blend_branches(gbuf[0], gbuf[1])]
        seen += np.array(shares)
        if kind != "smooth":  # each branch at each pos, so that theta and 1 - theta are told apart
            assert min(shares) > 0, shares
        # the scratch planes: within the any-order bound of the raw sums, carried through the normalisation
        con = im.splat(*planes[2:], pos, w, h, pitch)
        T = {p: im.terms(con[p], h * pitch) for p in im.PLANES}
        iv = im.normalised_intervals(T, corrected, w, h, pitch)
        skipped = np.zeros((h, w), bool)
        for k, name in enumerate(im.PLANES):
            lo, hi = iv[k]
            det = ~np.isnan(lo)
            skipped |= ~det
            g = gbuf[k].astype(np.float64)
            bad = det & ~((g >= lo) & (g <= hi))
            assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:3].tolist())
        print(f"{kind} {h}x{w} corrected={corrected} pos={pos}: {int(skipped.sum())} of {h * w} pixels "
              f"({skipped.mean():.2e}) not determined by the bound (a coverage interval contains 0); "
              f"branch pixel counts {shares}")
        assert skipped.mean() < 1e-3
        # the order matters here: not every accumulator is order-free
        assert not all(im.order_free(T[p]).all() for p in im.PLANES)
    assert seen.min() > 0, seen  # every blend branch was compared
