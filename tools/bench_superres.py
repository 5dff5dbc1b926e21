"""Time BTV-L1 super-resolution on the GPU (csrc/superres.cu) and write one JSON record.

    python tools/bench_superres.py [--out records/h100_superres.json] [--frames 6]

Two configurations:
  perf  the reference's perf test (modules/superres/perf/perf_superres.cpp:118-152): 128 x 128 8UC1 and 8UC3, scale 2,
        50 iterations, R = 1, zero flow, the same frame on every call; time per nextFrame in steady state;
  user  480 x 270 8UC3 -> 1920 x 1080 at the defaults (scale 4, 180 iterations, R = 4) with Farneback flows; time per
        output frame, split into the flows (two Farneback calls per frame) and the super-resolution itself.
Times come from CUDA events around whole nextFrame calls after a warm-up.  The record also holds launches per output
frame, the compulsory bytes of one iteration computed from shapes (see iteration_bytes), and the card's name and power
limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

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


def iteration_bytes(h, w, cn, s, K):
    """Compulsory bytes of one iteration, every buffer touched once: the forward pass reads hr (C floats per
    high-resolution pixel), the K backward maps (int32) and the K window frames, and writes K int8 sign planes; the update
    reads and writes hr and reads the K forward maps and the sign planes.  The blur taps and the BTV stencil re-read
    neighbours, which caches serve; they are not counted."""
    lr, hr = h * w, h * s * w * s
    fwd = hr * 4 * cn + K * hr * 4 + K * lr * 4 * cn + K * lr * cn
    upd = hr * 8 * cn + K * hr * 4 + K * lr * cn
    return float(fwd + upd)


class Zero:
    def __init__(self, h, w):
        import torch
        self.z = torch.zeros((h, w), dtype=torch.float32, device="cuda")

    def calc(self, f0, f1, u, v):
        return self.z, self.z


def run(sr, frames, n_out, warm):
    import torch
    sr.setInput(frames)
    for _ in range(warm):
        sr.nextFrame()
    torch.cuda.synchronize()
    sr.resetStats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_out):
        sr.nextFrame()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n_out, sr.getStats()["launches"] / n_out


def main():
    import torch
    import opencv_contrib_b200 as ocb

    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "records", "h100_superres.json"))
    ap.add_argument("--frames", type=int, default=6)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    rec = {"gpu": smi(), "perf": {}, "user": {}}

    for cn in (1, 3):
        frame = rng.integers(0, 256, (128, 128) + ((cn,) if cn > 1 else ()), dtype=np.uint8)
        frame_t = torch.from_numpy(frame).cuda()
        sr = ocb.createSuperResolution_BTVL1_CUDA()
        sr.setOpticalFlow(Zero(128, 128))
        sr.setScale(2), sr.setIterations(50), sr.setTemporalAreaRadius(1)
        ms, launches = run(sr, [frame_t] * (a.frames + 20), a.frames + 10, 5)
        rec["perf"][f"8UC{cn}"] = {"ms_per_next_frame": ms, "launches_per_output": launches,
                                   "iteration_compulsory_bytes": iteration_bytes(128, 128, cn, 2, 3)}

    h, w, R, warm = 270, 480, 4, 3
    n = a.frames
    # steady state: every timed output has the full 2R + 1 window and reads (and computes the flows of) a new frame,
    # so the stream holds 2R + 1 + warm + timed frames, and R more so no timed call reaches the end-of-stream flush
    count = 2 * R + 1 + warm + n + R
    base = rng.integers(0, 256, (h + 8, w + count, 3), dtype=np.uint8)
    frames = [torch.from_numpy(np.ascontiguousarray(base[t % 8:t % 8 + h, t:t + w])).cuda() for t in range(count)]
    sr = ocb.createSuperResolution_BTVL1_CUDA()
    ms, launches = run(sr, frames, n, warm)
    flow = ocb.createOptFlow_Farneback_CUDA()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):
        flow.calc(frames[0], frames[1], None, True)
    e0.record()
    for i in range(10):
        flow.calc(frames[i], frames[i + 1], None, True)
        flow.calc(frames[i + 1], frames[i], None, True)
    e1.record()
    torch.cuda.synchronize()
    flows_ms = e0.elapsed_time(e1) / 10
    rec["user"] = {"input": [h, w, 3], "output": [h * 4 - 14, w * 4 - 14, 3], "ms_per_output_frame": ms,
                   "flows_ms_per_frame": flows_ms, "super_resolution_ms_per_frame": ms - flows_ms,
                   "launches_per_output": launches, "iterations": 180, "K": 2 * R + 1, "frames_in_stream": count,
                   "timed_outputs": n, "iteration_compulsory_bytes": iteration_bytes(h, w, 3, 4, 2 * R + 1)}
    u = rec["user"]
    u["ms_per_iteration"] = u["super_resolution_ms_per_frame"] / 180
    u["iteration_compulsory_gbps"] = u["iteration_compulsory_bytes"] / (u["ms_per_iteration"] * 1e6)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=2)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
