"""Measure cudaimgproc's corner classes on one GPU and write records/h100_gftt.json.

CUDA events around >= 20 calls after warm-up give call times: compute (both criteria, 640x480 and 1080p, 8U), detect at
the defaults with minDistance 0 and 3, and a per-frame detect + SparsePyrLK step at 1080p; the host
cv2.goodFeaturesToTrack is the CPU comparator.  Kernel times come from a separate torch.profiler run, by kernel name:
the response kernel's bytes (8-bit read + float written) over its own time are set against the H100 SXM's 3.35 TB/s,
and the selection kernel's share of detect is its time over the sum of detect's kernels.  The card's name and power
limit are read in the same run.

    python tools/bench_gftt.py [--out records/h100_gftt.json] [--iters 50]
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


def _time(fn, iters, warm=5):
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


def _kernel_ms(fn, iters):
    """Mean device time per call of each of our kernels that `fn` launches, by name, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("k_corner_response", "k_gftt_candidates", "k_gftt_select", "k_gftt_reset"):
            if name in e.key:
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                out[name] = out.get(name, 0.0) + t / 1e3 / iters
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import cv2
    import torch
    import opencv_contrib_b200 as ocb
    from oracle import synth
    dev = torch.device("cuda:0")
    rec = dict(card=_card(), iters=a.iters, results={})
    R = rec["results"]
    for rows, cols in ((480, 640), (1080, 1920)):
        img = np.clip(np.rint(synth.texture(rows, cols, 1)), 0, 255).astype(np.uint8)
        d = torch.from_numpy(img).to(dev)
        out = torch.empty((rows, cols), dtype=torch.float32, device=dev)
        for name, crit in (("mineig", ocb.createMinEigenValCorner(0, 3, 3)), ("harris", ocb.createHarrisCorner(0, 3, 3, 0.04))):
            R[f"compute_{name}_{cols}x{rows}_call_ms"] = _time(lambda: crit.compute(d, out), a.iters)
            k = _kernel_ms(lambda: crit.compute(d, out), a.iters)
            kms = k.get("k_corner_response", float("nan"))
            R[f"compute_{name}_{cols}x{rows}_kernel_ms"] = kms
            R[f"compute_{name}_{cols}x{rows}_kernel_GBps"] = rows * cols * 5 / (kms * 1e-3) / 1e9
            R[f"compute_{name}_{cols}x{rows}_kernel_share_of_3350GBps"] = rows * cols * 5 / (kms * 1e-3) / 1e9 / 3350
    I0, I1, _ = synth.make_pair(1080, 1920, seed=3, kind="const")
    d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
    for md in (0.0, 3.0):
        det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, md)
        corners, count = det.detect_async(d0)
        R[f"detect_1080p_md{md:g}_ms"] = _time(lambda: det.detect_async(d0, corners=corners, count=count), a.iters)
        R[f"detect_1080p_md{md:g}_info"] = det.lastInfo()
        R[f"detect_1080p_md{md:g}_corners"] = int(count.item())
    for md in (0.0, 3.0):  # kernel times of one detect, from the profiler
        det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, md)
        corners, count = det.detect_async(d0)
        k = _kernel_ms(lambda: det.detect_async(d0, corners=corners, count=count), a.iters)
        R[f"detect_1080p_md{md:g}_kernel_ms"] = k
        R[f"detect_1080p_md{md:g}_selection_share_of_kernel_time"] = k.get("k_gftt_select", 0.0) / sum(k.values())
    det = ocb.createGoodFeaturesToTrackDetector(0, 1000, 0.01, 3.0)
    lk = ocb.SparsePyrLKOpticalFlow_create()

    def step():
        pts = det.detect(d0)
        lk.calc(d0, d1, pts)
    R["detect_plus_sparselk_1080p_ms"] = _time(step, max(20, a.iters // 2))
    t = time.perf_counter()
    n = 10
    for _ in range(n):
        cv2.goodFeaturesToTrack(I0, 1000, 0.01, 3.0)
    R["cpu_cv2_goodFeaturesToTrack_1080p_md3_ms"] = (time.perf_counter() - t) / n * 1e3
    R["cpu_threads"] = cv2.getNumThreads()
    rec["note"] = ("The reference's CUDA detector is not measured: it needs a CUDA build of OpenCV core, which this "
                   "project does not have.")
    js = json.dumps(rec, indent=1, default=str)
    print(js)
    if a.out:
        with open(a.out, "w") as f:
            f.write(js + "\n")


if __name__ == "__main__":
    main()
