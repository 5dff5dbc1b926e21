"""DeepFlow throughput: pairs/s on one GPU, device-resident, on one stream and through b2f_batch with N streams, at
640x480 and 1920x1080 on seeded synthetic u8 pairs (oracle/synth.py).  Prints one JSON line.

Alongside the rates:
  * sor_gbps -- the SOR solver's algorithmic bytes over its event time, from one profiled (graph-less) pair.  The
    algorithmic traffic of one SOR iteration is 44 B/px: the seven per-cell constants (a12, b1, b2, den_u, den_v and the
    right / lower edge weights) and (du, dv) read once, (du, dv) written once; a level that fits one region also counts
    its system terms (88 B/px per fixed-point step) in this class;
  * launches_per_pair -- kernel launches of one pair (all captured in one CUDA graph);
  * cpu_s_per_pair -- oracle/deepflow_ref.py (the reference's driver over cv2.VariationalRefinement) on this host's
    CPUs, with cv2's thread count;
  * gpu_name and power_limit_w, read in the same run.

    python tools/bench_deepflow.py [--pairs 8] [--streams 4] [--cpu-reps 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import opencv_contrib_b200 as ocb  # noqa: E402
from opencv_contrib_b200.batch import NativeFlowBatch  # noqa: E402
from oracle import synth, deepflow_ref  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=8)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--cpu-reps", type=int, default=1)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    import cv2
    rec = {"metric": "DeepFlow frame-pairs/sec", "gpu_name": torch.cuda.get_device_name(0),
           "power_limit_w": power_limit_w(), "cv2": cv2.__version__, "cv2_threads": cv2.getNumThreads(),
           "params": "createOptFlow_DeepFlow defaults", "sizes": {}}
    for h, w in ((480, 640), (1080, 1920)):
        frames = [synth.make_pair(h, w, seed=s, kind="smooth")[0] for s in range(args.pairs + 1)]
        dframes = [torch.from_numpy(f).to(dev) for f in frames]
        flows = [torch.empty((h, w, 2), dtype=torch.float32, device=dev) for _ in range(args.pairs)]
        alg = ocb.createOptFlow_DeepFlow()
        s = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(s):
            alg.calc(dframes[0], dframes[1], flows[0], stream=s)  # capture
            s.synchronize()
            alg.resetStats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for i in range(args.pairs):
                alg.calc(dframes[i], dframes[i + 1], flows[i], stream=s)
            e1.record(s)
        e1.synchronize()
        one_ms = e0.elapsed_time(e1) / args.pairs
        launches = alg.getStats()["launches"] / args.pairs

        nb = NativeFlowBatch("deepflow", None, n_streams=args.streams)
        pairs = [(dframes[i], dframes[i + 1]) for i in range(args.pairs)]
        nb.run_device(pairs, flows, stream=s)  # warm-up: workspaces and graphs
        s.synchronize()
        e0.record(s)
        nb.run_device(pairs, flows, stream=s)
        e1.record(s)
        e1.synchronize()
        batch_ms = e0.elapsed_time(e1) / args.pairs
        nb.close()

        prof = ocb.createOptFlow_DeepFlow()
        prof.setProfiling(True)
        prof.calc(dframes[0], dframes[1], flows[0])
        torch.cuda.synchronize()
        sor = prof.getStats()["classes"]["deepflow_sor"]

        t = time.perf_counter()
        for _ in range(args.cpu_reps):
            deepflow_ref.calc(frames[0], frames[1])
        cpu_s = (time.perf_counter() - t) / args.cpu_reps
        rec["sizes"]["%dx%d" % (w, h)] = {
            "levels": len(deepflow_ref.pyramid_sizes(h, w)),
            "pairs_per_s_1stream": 1000.0 / one_ms, "ms_per_pair_1stream": one_ms,
            "pairs_per_s_batch": 1000.0 / batch_ms, "batch_streams": args.streams,
            "launches_per_pair": launches,
            "sor_ms_per_pair_profiled": sor["ms"], "sor_gbps": sor["bytes"] / (sor["ms"] * 1e-3) / 1e9,
            "cpu_s_per_pair": cpu_s}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
