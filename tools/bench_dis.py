"""DIS throughput: pairs/s per preset on one GPU, device-resident, on one stream and through b2f_batch with N streams, at
640x480 and 1920x1080 on seeded synthetic u8 pairs with known smooth motion (oracle/synth.py).  Prints one JSON line.

Alongside the rates:
  * launches_per_pair -- kernel launches of one pair (all but the finest-level resize and the output interleave are
    captured in one CUDA graph);
  * class_ms -- per kernel class (scan, descent, densification, refinement, pyramid) the event time of one profiled
    (graph-less) pair;
  * cpu_ms_per_pair -- cv2.DISOpticalFlow with the same preset on this host's CPUs, with cv2's thread count;
  * gpu_name and power_limit_w, read in the same run.

    python tools/bench_dis.py [--pairs 16] [--streams 4] [--cpu-reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import opencv_contrib_b200 as ocb  # noqa: E402
from opencv_contrib_b200 import _lib  # noqa: E402
from opencv_contrib_b200.batch import NativeFlowBatch  # noqa: E402
from oracle import synth  # noqa: E402

PRESETS = {"ultrafast": 0, "fast": 1, "medium": 2}


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 - reported as unknown
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--cpu-reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    import cv2
    rec = {"metric": "DIS frame-pairs/sec", "gpu_name": torch.cuda.get_device_name(0),
           "power_limit_w": power_limit_w(), "cv2": cv2.__version__, "cv2_threads": cv2.getNumThreads(), "sizes": {}}
    for h, w in ((480, 640), (1080, 1920)):
        # each pair is one synthetic pair with known smooth motion (not two unrelated frames): the descents' early
        # stops depend on the content, so the pairs must be related as video frames are
        host = [synth.make_pair(h, w, seed=k, kind="smooth")[:2] for k in range(args.pairs)]
        pairs = [tuple(torch.from_numpy(f).to(dev) for f in pr) for pr in host]
        flows = [torch.empty((h, w, 2), dtype=torch.float32, device=dev) for _ in range(args.pairs)]
        per = {}
        for name, preset in PRESETS.items():
            alg = ocb.DISOpticalFlow_create(preset)
            s = torch.cuda.Stream(device=dev)
            with torch.cuda.stream(s):
                alg.calc(*pairs[0], flows[0], stream=s)  # capture
                s.synchronize()
                alg.resetStats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                for i in range(args.pairs):
                    alg.calc(*pairs[i], flows[i], stream=s)
                e1.record(s)
            e1.synchronize()
            one_ms = e0.elapsed_time(e1) / args.pairs
            launches = alg.getStats()["launches"] / args.pairs

            p = _lib.b2f_dis_params()
            _lib.lib().b2f_dis_default_params(p, preset)
            nb = NativeFlowBatch("dis", {k: getattr(p, k) for k, _ in p._fields_}, n_streams=args.streams)
            nb.run_device(pairs, flows, stream=s)  # warm-up: workspaces and graphs
            s.synchronize()
            e0.record(s)
            nb.run_device(pairs, flows, stream=s)
            e1.record(s)
            e1.synchronize()
            batch_ms = e0.elapsed_time(e1) / args.pairs
            nb.close()

            prof = ocb.DISOpticalFlow_create(preset)
            prof.setProfiling(True)
            prof.calc(*pairs[0], flows[0])
            torch.cuda.synchronize()
            classes = {k: round(v["ms"], 4) for k, v in prof.getStats()["classes"].items()}

            d = cv2.DISOpticalFlow_create(preset)
            d.calc(*host[0], None)
            t = time.perf_counter()
            for _ in range(args.cpu_reps):
                d.calc(*host[0], None)
            cpu_ms = (time.perf_counter() - t) / args.cpu_reps * 1e3
            per[name] = {"pairs_per_s_1stream": 1000.0 / one_ms, "ms_per_pair_1stream": one_ms,
                         "pairs_per_s_batch": 1000.0 / batch_ms, "batch_streams": args.streams,
                         "launches_per_pair": launches, "class_ms_profiled": classes, "cpu_ms_per_pair": cpu_ms}
        rec["sizes"]["%dx%d" % (w, h)] = per
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
