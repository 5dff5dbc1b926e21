"""VariationalRefinement throughput on one GPU, device-resident: ms per call on one stream and through b2f_batch with N
streams, at 640x480, 1920x1080 and 3840x2160, with (fixed-point, SOR) iterations (5, 5) -- cv2's defaults -- and
(5, 25), on seeded synthetic u8 pairs with known smooth motion (oracle/synth.py), each call refining the true flow
perturbed by up to 1 px.  Prints one JSON line and writes it to --out.

Alongside the times:
  * algorithmic_bytes_per_call and achieved_gbps -- per pixel warp 32 B + derivatives 36 B + per fixed-point step
    (system terms 88 B + 44 B per SOR iteration) + the add 24 B, over the one-stream time; the conversion, split and
    merge around the solver are not counted;
  * launches_per_call, and class_ms of one profiled (graph-less) call;
  * farneback_then_varref_1080p -- cv::cuda::FarnebackOpticalFlow (defaults) then VariationalRefinement (defaults) on
    one stream, per pair, against Farneback alone;
  * cpu_ms_per_call -- cv2.VariationalRefinement with the same iterations on this host's CPUs, with cv2's thread count;
  * gpu_name and power_limit_w, read in the same run.

    python tools/bench_varref.py [--calls 20] [--streams 4] [--cpu-reps 2] [--out records/h100_varref.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import opencv_contrib_b200 as ocb  # noqa: E402
from opencv_contrib_b200.batch import NativeFlowBatch  # noqa: E402
from oracle import synth  # noqa: E402

SIZES = ((480, 640), (1080, 1920), (2160, 3840))
ITERS = ((5, 5), (5, 25))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def algorithmic_bytes(h, w, fp, sor):
    return h * w * (32.0 + 36.0 + fp * (88.0 + 44.0 * sor) + 24.0)


def case(h, w, seed):
    I0, I1, gt = synth.make_pair(h, w, seed=seed, kind="smooth")
    rng = np.random.default_rng(seed)
    return I0, I1, (gt + (rng.random(gt.shape) - 0.5) * 2).astype(np.float32)


def make(fp, sor):
    alg = ocb.VariationalRefinement_create()
    alg.setFixedPointIterations(fp)
    alg.setSorIterations(sor)
    return alg


def timed(s, n, body):
    """ms per iteration of `body` over n iterations on stream s, by CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(n):
        body()
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--cpu-reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_varref.json"))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    import cv2
    rec = {"metric": "VariationalRefinement ms per call", "gpu_name": torch.cuda.get_device_name(0),
           "power_limit_w": power_limit_w(), "cv2": cv2.__version__, "cv2_threads": cv2.getNumThreads(),
           "calls": args.calls, "sizes": {}}
    s = torch.cuda.Stream(device=dev)
    for h, w in SIZES:
        host = [case(h, w, k) for k in range(args.streams)]
        pairs = [(torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)) for a, b, _ in host]
        flows = [torch.from_numpy(f).to(dev) for _, _, f in host]
        per = {}
        for fp, sor in ITERS:
            alg = make(fp, sor)
            with torch.cuda.stream(s):
                for _ in range(3):  # workspace, graph capture, warm
                    alg.calc(*pairs[0], flows[0], stream=s)
                s.synchronize()
                alg.resetStats()
                one_ms = timed(s, args.calls, lambda: alg.calc(*pairs[0], flows[0], stream=s))
            launches = alg.getStats()["launches"] / args.calls

            nb = NativeFlowBatch("varref", dict(fixed_point_iterations=fp, sor_iterations=sor), n_streams=args.streams)
            nb.run_device(pairs, flows, stream=s)  # workspaces and graphs
            s.synchronize()
            reps = max(1, args.calls // args.streams)
            batch_ms = timed(s, reps, lambda: nb.run_device(pairs, flows, stream=s)) / args.streams
            nb.close()

            prof = make(fp, sor)
            prof.setProfiling(True)
            prof.calc(*pairs[0], flows[0])
            torch.cuda.synchronize()
            classes = {k: round(v["ms"], 4) for k, v in prof.getStats()["classes"].items()}

            vr = cv2.VariationalRefinement_create()
            vr.setFixedPointIterations(fp)
            vr.setSorIterations(sor)
            a, b, f = host[0]
            vr.calc(a, b, f.copy())
            t = time.perf_counter()
            for _ in range(args.cpu_reps):
                vr.calc(a, b, f.copy())
            cpu_ms = (time.perf_counter() - t) / args.cpu_reps * 1e3
            nbytes = algorithmic_bytes(h, w, fp, sor)
            per["fp%d_sor%d" % (fp, sor)] = {
                "ms_per_call_1stream": one_ms, "ms_per_call_batch": batch_ms, "batch_streams": args.streams,
                "sor_iterations_per_launch": alg.getActivePath(), "launches_per_call": launches,
                "algorithmic_bytes_per_call": nbytes, "achieved_gbps": nbytes / (one_ms * 1e-3) / 1e9,
                "class_ms_profiled": classes, "cpu_ms_per_call": cpu_ms}
        rec["sizes"]["%dx%d" % (w, h)] = per

    h, w = 1080, 1920
    a, b, f = case(h, w, 0)
    d0, d1 = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
    flow = torch.empty((h, w, 2), dtype=torch.float32, device=dev)
    farn, vr = ocb.FarnebackOpticalFlow_create(), ocb.VariationalRefinement_create()

    def both():
        farn.calc(d0, d1, flow, stream=s)
        vr.calc(d0, d1, flow, stream=s)

    with torch.cuda.stream(s):
        for _ in range(3):
            both()
        s.synchronize()
        farn_ms = timed(s, args.calls, lambda: farn.calc(d0, d1, flow, stream=s))
        both_ms = timed(s, args.calls, both)
    rec["farneback_then_varref_1080p"] = {"farneback_ms": farn_ms, "farneback_then_varref_ms": both_ms}
    line = json.dumps(rec)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        fh.write(line + "\n")


if __name__ == "__main__":
    main()
