"""Time cudalegacy's block-matching flows on the GPU (csrc/bm.cu) and write one JSON record.

    python tools/bench_bm.py [--out records/h100_bm.json] [--reps 20]

FastOpticalFlowBM at 640x480 and 1080p for (search_window, block_window) = (21, 7) and (41, 9), on one stream and
through b2f_batch with 4 streams; calcOpticalFlowBM at 1080p (block 16x16, shift 8x8, range 16x16), cold and with
use_previous on the next pair; the numpy model's CPU time (a model, not a reference implementation).  The reference's
own GPU time is not measured: it needs a CUDA build of OpenCV core.  Times come from CUDA events around `reps` calls
after a warm-up; the card's name, power limit and SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def smi():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(smmax)}
    except Exception as e:  # noqa: BLE001 -- recorded, not fatal
        return {"error": str(e)}


def fastbm_ops(rows, cols, sw, bw):
    """Integer operations of a brute-force SAD search: per pixel and candidate, bw^2 absolute differences and adds,
    plus one compare.  The engine does fewer (sliding sums), so this is an equivalent rate, not an issued count."""
    return float(rows) * cols * sw * sw * (2 * bw * bw + 1)


def grid_ops(vr, vc, bw, bh, cands):
    return float(vr) * vc * cands * (2 * bw * bh + 1)


def time_cuda(fn, reps, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_bm.json"))
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    import opencv_contrib_b200 as ocb
    from opencv_contrib_b200.batch import NativeFlowBatch
    from oracle import bm_model, synth
    assert torch.cuda.is_available(), "bench_bm.py measures the GPU and needs one"
    props = torch.cuda.get_device_properties(0)
    card = smi()
    rec = {"gpu": card, "sm_count": props.multi_processor_count,
           "reference_gpu_time": "not measured (needs a CUDA build of OpenCV core)", "fastbm": [], "grid": []}
    clock_hz = card.get("sm_clock_max_mhz", 0) * 1e6
    int_bound = 64 * props.multi_processor_count * clock_hz  # INT32 lanes per SM per clock on Hopper
    rec["int32_issue_bound_ops_per_s"] = int_bound
    for rows, cols in ((480, 640), (1080, 1920)):
        I0, I1, _ = synth.make_pair(rows, cols, seed=0, kind="const")
        d0, d1 = torch.from_numpy(I0).cuda(), torch.from_numpy(I1).cuda()
        for sw, bw in ((21, 7), (41, 9)):
            alg = ocb.FastOpticalFlowBM(search_window=sw, block_window=bw)
            flow = torch.empty((rows, cols, 2), dtype=torch.float32, device="cuda")
            ms = time_cuda(lambda: alg.calc(d0, d1, flow), a.reps)
            nb = NativeFlowBatch("fastbm", dict(search_window=sw, block_window=bw), n_streams=4)
            pairs, flows = [(d0, d1)] * 8, [torch.empty_like(flow) for _ in range(8)]
            ms_b = time_cuda(lambda: nb.run_device(pairs, flows), max(2, a.reps // 4)) / 8
            assert np.array_equal(flow.cpu().numpy(), flows[0].cpu().numpy())
            ops = fastbm_ops(rows, cols, sw, bw)
            rec["fastbm"].append({"rows": rows, "cols": cols, "search_window": sw, "block_window": bw,
                                  "ms_one_stream": ms, "pairs_per_s_one_stream": 1e3 / ms,
                                  "ms_per_pair_batch4": ms_b, "pairs_per_s_batch4": 1e3 / ms_b,
                                  "bruteforce_equiv_int_ops_per_s": ops / (ms * 1e-3),
                                  "bruteforce_equiv_over_int32_bound": ops / (ms * 1e-3) / int_bound if int_bound else None})
            print(json.dumps(rec["fastbm"][-1]))
            if (rows, sw) == (480, 21):
                t = time.perf_counter()
                want = bm_model.fastbm(I0, I1, sw, bw)
                rec["numpy_model_fastbm_640x480_21_7_s"] = time.perf_counter() - t
                assert np.array_equal(flow.cpu().numpy(), want)
    I0, I1, _ = synth.make_pair(1080, 1920, seed=1, kind="const")
    J0, J1, _ = synth.make_pair(1080, 1920, seed=2, kind="const")
    d = [torch.from_numpy(x).cuda() for x in (I0, I1, J0, J1)]
    block, shift, rng_ = (16, 16), (8, 8), (16, 16)
    vr, vc = bm_model.vel_size(1080, 1920, block, shift)
    vx = torch.empty((vr, vc), dtype=torch.float32, device="cuda")
    vy = torch.empty_like(vx)
    ms_cold = time_cuda(lambda: ocb.calcOpticalFlowBM(d[0], d[1], block, shift, rng_, False, vx, vy), a.reps)
    gx, gy = ocb.calcOpticalFlowBM(d[0], d[1], block, shift, rng_, False)
    px, py = gx.clone(), gy.clone()

    def warm():
        vx.copy_(px)
        vy.copy_(py)
        ocb.calcOpticalFlowBM(d[2], d[3], block, shift, rng_, True, vx, vy)
    ms_copy = time_cuda(lambda: (vx.copy_(px), vy.copy_(py)), a.reps)
    ms_warm = time_cuda(warm, a.reps) - ms_copy
    c = {}
    t = time.perf_counter()
    want = bm_model.calc_bm(I0, I1, block, shift, rng_, False, counters=c)
    rec["numpy_model_grid_1080p_cold_s"] = time.perf_counter() - t
    assert np.array_equal(gx.cpu().numpy(), want[0]) and np.array_equal(gy.cpu().numpy(), want[1])
    cands = (2 * rng_[0] + 1) * (2 * rng_[1] + 1) - 1
    rec["grid"].append({"rows": 1080, "cols": 1920, "block": block, "shift": shift, "range": rng_, "vel_size": [vr, vc],
                        "ms_cold": ms_cold, "ms_use_previous_next_pair": ms_warm, "model_branches_cold": c,
                        "bruteforce_full_scan_int_ops": grid_ops(vr, vc, *block, cands)})
    print(json.dumps(rec["grid"][-1]))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps({"gpu": card, "out": a.out}))


if __name__ == "__main__":
    main()
