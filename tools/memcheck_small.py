"""Small-size pass over every engine and adjacent component (run under compute-sanitizer)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, cv2
import opencv_contrib_b200 as ocb
from oracle import synth
dev = torch.device("cuda:0")
I0, I1, _ = synth.make_pair(141, 203, seed=3, kind="smooth")
d0, d1 = torch.from_numpy(I0).to(dev), torch.from_numpy(I1).to(dev)
f0, f1 = d0.float() / 255, d1.float() / 255
for name, alg, a, b in [
        ("tvl1", ocb.OpticalFlowDual_TVL1_create(nscales=3, warps=2, epsilon=0.0, iterations=9), d0, d1),
        ("tvl1-eps", ocb.OpticalFlowDual_TVL1_create(nscales=2, warps=2, iterations=12), d0, d1),
        ("farneback", ocb.FarnebackOpticalFlow_create(numLevels=3, numIters=2), d0, d1),
        ("brox", ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 7), f0, f1),
        ("brox-pp", ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 3), f0, f1),
        ("brox-coop", ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 3, 10, 5), f0, f1),
        ("brox-exact-rsqrt", ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 4), f0, f1),
        ("denselk", ocb.DensePyrLKOpticalFlow_create(maxLevel=2, iters=4), d0, d1),
        ("denselk-generic", ocb.DensePyrLKOpticalFlow_create(winSize=(9, 7), maxLevel=1, iters=3), d0, d1),
        ("denselk-even", ocb.DensePyrLKOpticalFlow_create(winSize=(4, 6), maxLevel=1, iters=3), d0, d1),
        ("denselk-fast-even", ocb.DensePyrLKOpticalFlow_create(winSize=(13, 6), maxLevel=1, iters=3), d0, d1)]:
    if name == "brox-pp":
        alg.setEngineOption("kernel_path", 2)
    if name == "brox-coop":
        alg.setEngineOption("kernel_path", 3)
    if name == "brox-exact-rsqrt":
        alg.setEngineOption("aux_path", 1)
    if len(sys.argv) > 1 and not any(name.startswith(a) for a in sys.argv[1:]):
        continue
    alg.setEngineOption("use_graph", 0)
    fl = alg.calc(a, b, torch.zeros((141, 203, 2), device=dev))
    u, v = alg.calcUV(a, b, torch.zeros((141, 203), device=dev), torch.zeros((141, 203), device=dev))
    torch.cuda.synchronize()
    print(name, "ok", float(fl.abs().mean()), flush=True)
fl = fl.contiguous()
# Farneback iteration-kernel variants: (name, size, create() arguments, kernel_path, aux_path).  983 x 1053 has more than
# 2 x 132 64x64 tiles, so kernel_path 3 runs the persistent TMA kernel there; the other sizes have more than 132 64x32
# tiles at level 0 where the aux variants need it.
for name, (h, w), kw, kp, aux in [
        ("farneback-generic", (141, 203), dict(numLevels=2, numIters=2), 1, 0),
        ("farneback-pixel-gather", (141, 203), dict(numLevels=2, numIters=2, flags=256), 2, 0),
        ("farneback-tma", (983, 1053), dict(numLevels=0, numIters=2), 3, 0),
        ("farneback-aux3", (315, 933), dict(numLevels=1, numIters=2), 0, 3),
        ("farneback-aux4", (315, 933), dict(numLevels=1, numIters=2), 0, 4),
        ("farneback-aux5", (315, 933), dict(numLevels=1, numIters=2), 0, 5),
        ("farneback-win1", (141, 203), dict(numLevels=1, numIters=2, winSize=1), 0, 0),
        ("farneback-win31", (141, 203), dict(numLevels=1, numIters=2, winSize=31, flags=256), 0, 0),
        ("farneback-1x37", (1, 37), dict(numLevels=0, numIters=3), 0, 0),
        ("farneback-37x1", (37, 1), dict(numLevels=0, numIters=3, flags=256), 0, 0)]:
    if len(sys.argv) > 1 and not any(name.startswith(a) for a in sys.argv[1:]):
        continue
    J0, J1, _ = synth.make_pair(max(h, 16), max(w, 16), seed=5, kind="smooth")
    j0 = torch.from_numpy(np.ascontiguousarray(J0[:h, :w])).to(dev)
    j1 = torch.from_numpy(np.ascontiguousarray(J1[:h, :w])).to(dev)
    alg = ocb.FarnebackOpticalFlow_create(**kw)
    alg.setEngineOption("kernel_path", kp)
    alg.setEngineOption("aux_path", aux)
    alg.setEngineOption("use_graph", 0)
    ff = alg.calc(j0, j1)
    torch.cuda.synchronize()
    print(name, "ok", float(ff.abs().mean()), "active path", [alg.getActivePath(k) for k in range(alg.getStats()["levels"])],
          flush=True)
# Brox at the edge shapes of tests/test_brox_fullsize_gpu.py, every solver path, correctly rounded data-term rsqrt
for (h, w), kp in [((1, 37), 0), ((37, 1), 0), ((2, 2), 0), ((15, 200), 1), ((65, 63), 2), ((141, 203), 3)]:
    g = torch.rand((2, h, w), generator=torch.Generator().manual_seed(h * w)).to(dev)
    alg = ocb.BroxOpticalFlow_create(0.197, 50.0, 0.8, 2, 10, 3)
    alg.setEngineOption("kernel_path", kp)
    alg.setEngineOption("aux_path", 1)
    alg.setEngineOption("use_graph", 0)
    fb = alg.calc(g[0].contiguous(), g[1].contiguous())
    torch.cuda.synchronize()
    print("brox", (h, w), "kernel_path", kp, "ok", float(fb.abs().mean()), flush=True)
mid = ocb.interpolateFrames(f0, f1, fl[..., 0].contiguous(), fl[..., 1].contiguous(), -fl[..., 0].contiguous(),
                            -fl[..., 1].contiguous(), 0.3)
mid2 = ocb.interpolateFrames(f0, f1, fl[..., 0].contiguous(), fl[..., 1].contiguous(), -fl[..., 0].contiguous(),
                             -fl[..., 1].contiguous(), 0.3, corrected=True)
torch.cuda.synchronize()
print("interp ok", float(mid.mean()), float(mid2.mean()), flush=True)
pts = cv2.goodFeaturesToTrack(I0, 200, 0.01, 0.0).reshape(-1, 2).astype(np.float32)
sp = ocb.SparsePyrLKOpticalFlow_create(maxLevel=2, iters=8)
n, s, e = sp.calc(d0, d1, torch.from_numpy(pts).to(dev), wantErr=True)
torch.cuda.synchronize()
print("sparse ok", int(s.sum()), flush=True)
vf = ocb.VideoFlow(ocb.FarnebackOpticalFlow_create(numLevels=2, numIters=2), 141, 203, depth=2, warm_start=True)
out = list(vf.run([I0, I1, I0, I1, I0]))
vf.close()
print("video ok", len(out), flush=True)
