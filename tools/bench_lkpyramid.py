"""Measure the video module's calcOpticalFlowPyrLK on one GPU and write records/h100_lkpyramid.json.

CUDA events around repeated calls after warm-up give call times at 1080p (8UC1, 21 x 21 window, maxLevel 3, the default
criteria) for 2 000 GFTT points and 10 000 grid points, with both pyramids built inside the call and with pyramids
built beforehand and reused; buildOpticalFlowPyramid on its own; cv2.calcOpticalFlowPyrLK on the host's threads in the
same run.  The card's name and power limit are read in the same run.

    python tools/bench_lkpyramid.py [--out records/h100_lkpyramid.json] [--iters 30]
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


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(error=str(e))


def _time(fn, iters, warm=3):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    import cv2
    import torch
    from opencv_contrib_b200 import lkpyramid as LK
    from oracle import synth
    dev = torch.device("cuda:0")
    rec = dict(card=_card(), iters=a.iters, config="1080p 8UC1, winSize 21x21, maxLevel 3, criteria (COUNT|EPS, 30, 0.01)",
               results={})
    R = rec["results"]
    I0, I1, _ = synth.make_pair(1080, 1920, seed=3, kind="const")
    d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
    gf = cv2.goodFeaturesToTrack(I0, 2000, 0.01, 5).astype(np.float32)
    xs, ys = np.meshgrid(np.arange(10, 1910, 19.0), np.arange(10, 1070, 10.6))
    grid = np.stack([xs, ys], -1).reshape(-1, 1, 2)[:10000].astype(np.float32)
    lk = LK.SparsePyrLKOpticalFlow_create()
    _, p0 = LK.buildOpticalFlowPyramid(d0, (21, 21), 3)
    _, p1 = LK.buildOpticalFlowPyramid(d1, (21, 21), 3, withDerivatives=False)
    R["build_pyramid_with_derivatives_ms"] = _time(lambda: LK.buildOpticalFlowPyramid(d0, (21, 21), 3, p0), a.iters)
    R["build_pyramid_without_derivatives_ms"] = _time(
        lambda: LK.buildOpticalFlowPyramid(d1, (21, 21), 3, p1, withDerivatives=False), a.iters)
    for name, pts in (("gftt", gf), ("grid", grid)):
        n = len(pts)
        tp = torch.from_numpy(pts).to(dev)
        nxt = torch.empty_like(tp)
        st = torch.empty((n, 1), dtype=torch.uint8, device=dev)
        er = torch.zeros((n, 1), dtype=torch.float32, device=dev)
        R[f"{name}{n}_images_ms"] = _time(lambda: lk.calc(d0, d1, tp, nxt, st, er), a.iters)
        R[f"{name}{n}_pyramids_reused_ms"] = _time(lambda: lk.calc(p0, p1, tp, nxt, st, er), a.iters)
        # the frame loop a user writes: each new frame's pyramid is built once, into one of two rotating objects, and
        # tracked against the previous frame's (prev = nxt)
        bufs = [LK.buildOpticalFlowPyramid(d0, (21, 21), 3)[1], LK.buildOpticalFlowPyramid(d1, (21, 21), 3)[1]]
        step = [0]

        def loop():
            k = step[0] = step[0] + 1
            LK.buildOpticalFlowPyramid(d1 if k % 2 else d0, (21, 21), 3, bufs[k % 2])
            lk.calc(bufs[(k + 1) % 2], bufs[k % 2], tp, nxt, st, er)
        R[f"{name}{n}_frame_loop_build_plus_calc_ms"] = _time(loop, a.iters)
        R[f"{name}{n}_tracked"] = int(st.sum().item())
        k = 5
        t = time.perf_counter()
        for _ in range(k):
            cv2.calcOpticalFlowPyrLK(I0, I1, pts, None)
        R[f"{name}{n}_cpu_cv2_ms"] = (time.perf_counter() - t) / k * 1e3
    R["cpu_threads"] = cv2.getNumThreads()
    R["active_path"] = lk.getActivePath()
    js = json.dumps(rec, default=str)
    print(js)
    if a.out:
        with open(a.out, "w") as f:
            f.write(js + "\n")


if __name__ == "__main__":
    main()
