"""Round-2 TV-L1 probe, 1080p 5x10x30 eps=0: kernel_path x fused_iters sweep (single stream + 4 streams),
bit-equality against the unfused kernels, and the per-class launch-time breakdown of the default path."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import opencv_contrib_b200 as ocb
from oracle import synth
dev = torch.device("cuda:0")
I0, I1, gt = synth.make_pair(1080, 1920, seed=0, kind="smooth")
d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
ref = None
cases = [tuple(int(v) for v in (c.split(":") + ["0"])[:3]) for c in (sys.argv[1:] or ["0:8", "0:12"])]
for path, K, aux in cases:
    algs = [ocb.OpticalFlowDual_TVL1_create(nscales=5, warps=10, epsilon=0.0, iterations=30) for _ in range(4)]
    for a in algs:
        a.setEngineOption("fused_iters", K)
        a.setEngineOption("kernel_path", path)
        a.setEngineOption("aux_path", aux)
    flows = [torch.empty((1080, 1920, 2), dtype=torch.float32, device=dev) for _ in range(4)]
    streams = [torch.cuda.Stream() for _ in range(4)]
    for _ in range(2): algs[0].calc(d0, d1, flows[0])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 5
    e0.record()
    for _ in range(n): algs[0].calc(d0, d1, flows[0])
    e1.record(); torch.cuda.synchronize()
    ms1 = e0.elapsed_time(e1) / n
    out = flows[0].cpu().numpy()
    if ref is None: ref = out
    same = np.array_equal(out, ref)
    for i in range(4):
        with torch.cuda.stream(streams[i]): algs[i].calc(d0, d1, flows[i], streams[i])
    torch.cuda.synchronize()
    e0.record()
    for r in range(3):
        for i in range(4):
            if r == 0: streams[i].wait_event(e0)
            algs[i].calc(d0, d1, flows[i], streams[i])
    for s in streams: torch.cuda.current_stream().wait_stream(s)
    e1.record(); torch.cuda.synchronize()
    ms4 = e0.elapsed_time(e1) / 12
    a = algs[0]
    a.setProfiling(True); a.resetStats(); a.calc(d0, d1, flows[0]); torch.cuda.synchronize()
    st = a.getStats(); a.setProfiling(False)
    cls = ", ".join("%s %.2f ms/%d" % (k, v["ms"], v["launches"]) for k, v in st["classes"].items() if v["launches"])
    print("path=%d K=%d aux=%d: 1 stream %.2f ms/pair (%.1f/s); 4 streams %.2f ms/pair (%.1f/s); bit-equal to first: %s | %s"
          % (path, K, aux, ms1, 1000 / ms1, ms4, 1000 / ms4, same, cls), flush=True)
