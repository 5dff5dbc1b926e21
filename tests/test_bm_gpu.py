"""cudalegacy's block-matching flows on the GPU (csrc/bm.cu) against oracle/bm_model.py, bit for bit on the whole output:
FastOpticalFlowBM over frame sizes, the window grid, both key widths, tile-edge shapes, tiny frames, designed ties and
ROIs; calcOpticalFlowBM over block / shift / range sets, chained use_previous calls and its branches."""

import numpy as np
import pytest

from oracle import bm_model as M

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ocb():
    import opencv_contrib_b200 as m
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return m


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pair(rows, cols, seed=0, shift=(1, -2)):
    rng = np.random.default_rng(seed)
    I0 = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
    I1 = np.roll(I0, shift, (0, 1))
    noise = rng.random(I1.shape) < 0.1
    I1[noise] = rng.integers(0, 256, int(noise.sum()), dtype=np.uint8)
    return I0, I1


def run_fastbm(ocb, I0, I1, sw, bw):
    a = ocb.FastOpticalFlowBM()
    u, v = a(dev(I0), dev(I1), search_window=sw, block_window=bw)
    return np.stack([u.cpu().numpy(), v.cpu().numpy()], -1), a


def check(ocb, I0, I1, sw=21, bw=7):
    got, a = run_fastbm(ocb, I0, I1, sw, bw)
    want = M.fastbm(I0, I1, sw, bw)
    assert np.array_equal(got, want), (sw, bw, I0.shape, int((got != want).any(-1).sum()))
    return a


@pytest.mark.parametrize("shape,sw,bw", [((480, 640), 21, 7), ((1080, 1920), 21, 7), ((480, 640), 41, 9)])
def test_fastbm_frame_sizes(ocb, shape, sw, bw):
    I0, I1 = pair(*shape)
    check(ocb, I0, I1, sw, bw)


@pytest.mark.parametrize("sw", [1, 2, 21, 32, 109])
@pytest.mark.parametrize("bw", [1, 3, 7, 15, 31])
def test_fastbm_window_grid(ocb, sw, bw):
    I0, I1 = pair(70, 90, seed=sw + bw)
    I0, I1 = I0 // 64 * 64, I1 // 64 * 64  # coarse levels: many exact ties
    check(ocb, I0, I1, sw, bw)


@pytest.mark.parametrize("sw,bw", [(109, 21), (109, 23)])
def test_fastbm_both_key_widths(ocb, sw, bw):
    assert M.key_layout(109, 21)[1] is False and M.key_layout(109, 23)[1] is True
    I0, I1 = pair(80, 100, seed=4)
    a = check(ocb, I0, I1, sw, bw)
    assert a.getActivePath()[2] == M.key_layout(sw, bw)[1]


def test_fastbm_tile_edges(ocb):
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    ow, th, _ = run_fastbm(ocb, *pair(8, 8), 21, 7)[1].getActivePath()
    assert (ow, th) == (26, 64)
    for tiles in (n_sm, n_sm + 1, 2 * n_sm + 1):
        for extra in range(4):
            cols = ow * tiles + extra  # widths 0-3 mod 4 around the tile count
            I0, I1 = pair(th + 3, cols, seed=tiles + extra)
            check(ocb, I0, I1)


@pytest.mark.parametrize("shape", [(1, 1), (1, 37), (37, 1), (5, 5)])
def test_fastbm_border_exceeds_frame(ocb, shape):
    I0, I1 = pair(*shape, seed=7, shift=(0, 0))
    check(ocb, I0, I1)
    check(ocb, I0, I1, 109, 31)


def test_fastbm_flat_ties_and_max_sad(ocb):
    flat = np.full((40, 50), 9, np.uint8)
    got, _ = run_fastbm(ocb, flat, flat, 21, 7)
    assert (got == -10).all()
    from test_bm_model_cpu import tie_frames, TIE_SHIFT
    I0, I1 = tie_frames(21, 7, TIE_SHIFT)
    check(ocb, I0, I1, 21, 3)
    yy, xx = np.mgrid[:90, :120]
    board = ((yy + xx) % 2 * 255).astype(np.uint8)
    check(ocb, board, 255 - board, 109, 31)
    check(ocb, board, 255 - board, 109, 21)


def test_fastbm_rois_calc_and_calc_uv(ocb):
    I0, I1 = pair(101, 203, seed=9)
    big0 = torch.zeros((120, 333), dtype=torch.uint8, device="cuda")
    big1 = torch.zeros((117, 301), dtype=torch.uint8, device="cuda")
    r0, r1 = big0[5:106, 7:210], big1[3:104, 13:216]  # odd byte offsets and pitches
    r0.copy_(dev(I0))
    r1.copy_(dev(I1))
    a = ocb.FastOpticalFlowBM()
    u, v = a(r0, r1)
    want = M.fastbm(I0, I1)
    assert np.array_equal(np.stack([u.cpu().numpy(), v.cpu().numpy()], -1), want)
    assert np.array_equal(a.calc(r0, r1).cpu().numpy(), want)
    assert a.getStats()["classes"]["fastbm"]["launches"] == 2
    assert a.getDefaultName() == "DenseOpticalFlow.FastOpticalFlowBM"


def test_fastbm_handles_on_streams_and_batch(ocb):
    from opencv_contrib_b200.batch import NativeFlowBatch
    pairs = [pair(64, 96, seed=s) for s in range(6)]
    want = [M.fastbm(a, b) for a, b in pairs]
    algs = [ocb.FastOpticalFlowBM() for _ in range(3)]
    streams = [torch.cuda.Stream() for _ in range(3)]
    d = [(dev(a), dev(b)) for a, b in pairs]
    torch.cuda.synchronize()
    outs = [algs[i % 3].calc(a, b, stream=streams[i % 3]) for i, (a, b) in enumerate(d)]
    torch.cuda.synchronize()
    for o, w in zip(outs, want):
        assert np.array_equal(o.cpu().numpy(), w)
    nb = NativeFlowBatch("fastbm", n_streams=4)
    flows = [torch.empty((64, 96, 2), dtype=torch.float32, device="cuda") for _ in d]
    nb.run_device(d, flows)
    torch.cuda.synchronize()
    for o, w in zip(flows, want):
        assert np.array_equal(o.cpu().numpy(), w)


def test_fastbm_refusals(ocb):
    from opencv_contrib_b200._lib import B2FError
    I0, I1 = pair(20, 30)
    a = ocb.FastOpticalFlowBM()
    for sw, bw in ((21, 8), (110, 7), (0, 7), (21, 33), (21, 0), (21, -1)):
        with pytest.raises(B2FError) as e:
            a(dev(I0), dev(I1), search_window=sw, block_window=bw)
        assert e.value.status == 1, (sw, bw)
    with pytest.raises(B2FError) as e:
        a(dev(I0).float(), dev(I1).float())
    assert e.value.status == 2
    with pytest.raises(B2FError) as e:
        a(dev(I0), dev(I1[:, :29]))
    assert e.value.status == 3


# ------------------------------------------------------------------------------------------------ grid BM
def grid(ocb, prev, curr, block, shift, rng_, use_prev=False, vx=None, vy=None):
    gx, gy = ocb.calcOpticalFlowBM(dev(prev), dev(curr), block, shift, rng_, use_prev,
                                   None if vx is None else dev(vx), None if vy is None else dev(vy))
    return gx.cpu().numpy(), gy.cpu().numpy()


def check_grid(ocb, prev, curr, block, shift, rng_, use_prev=False, vx=None, vy=None):
    c = {}
    want = M.calc_bm(prev, curr, block, shift, rng_, use_prev, vx, vy, counters=c)
    got = grid(ocb, prev, curr, block, shift, rng_, use_prev, vx, vy)
    assert np.array_equal(got[0].view(np.int32), want[0].view(np.int32)), (block, shift, rng_)
    assert np.array_equal(got[1].view(np.int32), want[1].view(np.int32)), (block, shift, rng_)
    return got, c


GRID_CASES = [((8, 8), (8, 8), (4, 4)), ((16, 16), (8, 8), (3, 6)), ((16, 8), (4, 8), (6, 3)), ((8, 8), (4, 4), (0, 0)),
              ((5, 7), (9, 3), (2, 5)), ((7, 5), (3, 11), (5, 0))]


@pytest.mark.parametrize("block,shift,rng_", GRID_CASES)
def test_grid_sets(ocb, block, shift, rng_):
    for rows, cols in ((61, 83), (64, 96)):  # velSize remainders non-zero and zero for 8x8
        prev, curr = pair(rows, cols, seed=rows)
        check_grid(ocb, prev, curr, block, shift, rng_)
        noisy = np.random.default_rng(2).integers(0, 256, prev.shape, dtype=np.uint8)
        check_grid(ocb, prev, (prev // 2 + noisy // 2).astype(np.uint8), block, shift, rng_)


def test_grid_use_previous_chain(ocb):
    prev, curr = pair(72, 88, seed=3, shift=(2, -3))
    block, shift, rng_ = (8, 8), (8, 8), (3, 3)
    vr, vc = M.vel_size(72, 88, block, shift)
    vx = np.random.default_rng(1).uniform(-4, 4, (vr, vc)).astype(np.float32)
    vy = np.full((vr, vc), 0.5, np.float32)
    vx[0, :4] = [0.5, 1.5, -2.5, 3e9]
    vy[1, :3] = [np.nan, -1e12, 1e12]
    vx[2, 0] = 500.0  # out of range
    for _ in range(3):
        (gx, gy), _ = check_grid(ocb, prev, curr, block, shift, rng_, True, vx, vy)
        vx, vy = gx, gy


def test_grid_1080p(ocb):
    prev, curr = pair(1080, 1920, seed=11, shift=(3, -4))
    (gx, gy), c = check_grid(ocb, prev, curr, (16, 16), (8, 8), (16, 16))
    check_grid(ocb, prev, curr, (16, 16), (8, 8), (16, 16), True, gx, gy)


def test_grid_branches(ocb):
    from test_bm_model_cpu import branch_case
    for name in M.BRANCHES:
        p, q, use_prev, vel = branch_case(name)
        _, c = check_grid(ocb, p, q, (16, 16), (8, 8), (3, 3), use_prev, *(vel or (None, None)))
        assert c[name] > 0, (name, c)


def test_grid_rois_and_refusals(ocb):
    from opencv_contrib_b200._lib import B2FError
    prev, curr = pair(50, 70, seed=5)
    big = torch.zeros((60, 99), dtype=torch.uint8, device="cuda")
    big2 = torch.zeros((55, 91), dtype=torch.uint8, device="cuda")
    r0, r1 = big[3:53, 5:75], big2[1:51, 9:79]
    r0.copy_(dev(prev))
    r1.copy_(dev(curr))
    vx = torch.zeros((9, 21), dtype=torch.float32, device="cuda")
    vy = torch.zeros((9, 21), dtype=torch.float32, device="cuda")
    gx, gy = ocb.calcOpticalFlowBM(r0, r1, (8, 8), (8, 8), (3, 3), False, vx[1:7, 2:10], vy[2:8, 1:9])
    want = M.calc_bm(prev, curr, (8, 8), (8, 8), (3, 3), False)
    assert np.array_equal(gx.cpu().numpy(), want[0]) and np.array_equal(gy.cpu().numpy(), want[1])
    d0, d1 = dev(prev), dev(curr)
    for args, code in (((d0.float(), d1.float(), (8, 8), (8, 8), (3, 3), False), 2),
                       ((d0, d1[:, :60], (8, 8), (8, 8), (3, 3), False), 3),
                       ((d0, d1, (0, 8), (8, 8), (3, 3), False), 1), ((d0, d1, (8, 8), (8, 0), (3, 3), False), 1),
                       ((d0, d1, (8, 8), (8, 8), (-1, 3), False), 1), ((d0, d1, (71, 8), (8, 8), (3, 3), False), 1)):
        with pytest.raises(B2FError) as e:
            ocb.calcOpticalFlowBM(*args)
        assert e.value.status == code, args
    with pytest.raises(B2FError) as e:
        ocb.calcOpticalFlowBM(d0, d1, (8, 8), (8, 8), (3, 3), True, vx, vy)  # not of velSize
    assert e.value.status == 3
