"""The video module's Farneback engine (csrc/optflowgf.cu) on one GPU, device-resident: ms per pair on one stream and
pairs/s through b2f_batch with N streams, at 640x480 and 1920x1080, box and gaussian windows, cv2's default parameters
(0.5, 5, 13, 10, 5, 1.1), on seeded synthetic u8 pairs (oracle/synth.py).  In the same run: the cv::cuda Farneback
engine on the same pairs, default cv2 on this host's CPUs (cv2's thread count), and the card's name and power limit.
Prints one JSON line and writes it to --out.

    python tools/bench_optflowgf.py [--calls 20] [--streams 4] [--cpu-reps 3] [--out records/h100_optflowgf.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

import opencv_contrib_b200 as ocb  # noqa: E402
from opencv_contrib_b200 import optflowgf  # noqa: E402
from opencv_contrib_b200.batch import NativeFlowBatch  # noqa: E402
from oracle import synth  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, watts = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(watts)


def time_stream(alg, d0, d1, calls):
    s = torch.cuda.Stream()
    flow = torch.empty((d0.shape[0], d0.shape[1], 2), dtype=torch.float32, device="cuda")
    for _ in range(3):
        alg.calc(d0, d1, flow, stream=s)
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(calls):
        alg.calc(d0, d1, flow, stream=s)
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def time_batch(flags, d0, d1, streams, calls):
    nb = NativeFlowBatch("optflowgf", dict(flags=flags), n_streams=streams)
    pairs = [(d0, d1)] * (streams * 2)
    flows = [torch.empty((d0.shape[0], d0.shape[1], 2), dtype=torch.float32, device="cuda") for _ in pairs]
    nb.run_device(pairs, flows)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(max(1, calls // len(pairs))):
        nb.run_device(pairs, flows)
    torch.cuda.synchronize()
    n = max(1, calls // len(pairs)) * len(pairs)
    rate = n / (time.perf_counter() - t)
    nb.close()
    return rate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--cpu-reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_optflowgf.json"))
    a = ap.parse_args()
    name, watts = gpu_info()
    rec = {"gpu_name": name, "power_limit_w": watts, "params": [0.5, 5, 13, 10, 5, 1.1], "cpu_threads": cv2.getNumThreads(),
           "results": {}}
    for rows, cols in [(480, 640), (1080, 1920)]:
        I0, I1, _ = synth.make_pair(rows, cols, seed=0, kind="smooth")
        d0, d1 = torch.from_numpy(I0).cuda(), torch.from_numpy(I1).cuda()
        for win, flags in [("box", 0), ("gaussian", 256)]:
            key = f"{cols}x{rows}_{win}"
            gf = optflowgf.FarnebackOpticalFlow_create(flags=flags)
            cu = ocb.FarnebackOpticalFlow_create(flags=flags)
            r = {"optflowgf_ms_per_pair": time_stream(gf, d0, d1, a.calls),
                 "optflowgf_batch_pairs_per_s": time_batch(flags, d0, d1, a.streams, a.calls * a.streams),
                 "batch_streams": a.streams,
                 "cuda_farneback_ms_per_pair": time_stream(cu, d0, d1, a.calls)}
            ts = []
            for _ in range(a.cpu_reps):
                t = time.perf_counter()
                cv2.calcOpticalFlowFarneback(I0, I1, None, 0.5, 5, 13, 10, 5, 1.1, flags)
                ts.append((time.perf_counter() - t) * 1e3)
            r["cv2_default_ms_per_pair"] = ts
            rec["results"][key] = r
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
