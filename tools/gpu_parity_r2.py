"""Measured values behind the round-2 full-size / golden-vector parity tests: the same comparisons
the tests make, printed instead of asserted."""
import sys, os, importlib.util
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import synth, metrics, tvl1_cpu


def load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m); return m


T, B = load("test_tvl1_gpu"), load("test_brox_lk_gpu")
dev = torch.device("cuda:0")
fmt = lambda st: ", ".join("%s %.3g" % (k, v) for k, v in st.items())
for (h, w, name) in ((1080, 1920, "1080p"), (2160, 3840, "4K")):
    I0, I1, gt = synth.make_pair(h, w, seed=0, kind="smooth")
    got, _ = T._run(dev, I0, I1, nscales=5, warps=10, epsilon=0.0, iterations=30)
    cpu, kind = T._cpu_reference(I0, I1, tvl1_cpu.TVL1Params(nscales=5, warps=10, epsilon=0.0, innerIterations=1,
                                                           outerIterations=30, medianFiltering=1))
    st = metrics.epe_stats(got, cpu, border=32)
    ncc = metrics.ncc_dissimilarity(got[32:-32, 32:-32], cpu[32:-32, 32:-32])
    g_gpu, g_cpu = metrics.epe_stats(got, gt, border=32), metrics.epe_stats(cpu, gt, border=32)
    print("TV-L1 %s 5x10x30 eps=0 vs CPU %s: %s, NCC dissimilarity %.3g; mean EPE vs ground truth: GPU %.4f, CPU %.4f"
          % (name, kind, fmt(st), ncc, g_gpu["mean"], g_cpu["mean"]), flush=True)
gold = os.path.join(ROOT, "tests", "golden")
for name in sorted(os.listdir(gold)):
    if not (name.startswith("tvl1_ref_") and name.endswith(".npz")): continue
    z = np.load(os.path.join(gold, name))
    kw = {k[3:]: z[k].item() for k in z.files if k.startswith("kw_")}
    P = tvl1_cpu.TVL1Params(**kw)
    if P.epsilon > 0: continue
    got, _ = T._run(dev, z["I0"], z["I1"], nscales=P.nscales, warps=P.warps, epsilon=0.0,
                    iterations=P.innerIterations * P.outerIterations, gamma=P.gamma, _median=(P.medianFiltering, P.innerIterations))
    st = metrics.epe_stats(got, z["flow"], border=16)
    ncc = metrics.ncc_dissimilarity(got[16:-16, 16:-16], z["flow"][16:-16, 16:-16])
    print("TV-L1 golden %s (%s): %s, NCC dissimilarity %.3g" % (name, ", ".join("%s=%s" % kv for kv in kw.items()), fmt(st), ncc), flush=True)
from oracle import denselk_model_native as lkn  # noqa: E402
I0, I1, _ = synth.make_pair(1080, 1920, seed=0, kind="smooth")
got, _ = B._lk(dev, I0, I1, winSize=(13, 13), maxLevel=3, iters=30)
want = lkn.calc(I0, I1, (13, 13), 3, 30)
print("DensePyrLK 1080p defaults vs the C model: %d pixels differ" % int((got != want).any(axis=-1).sum()), flush=True)
