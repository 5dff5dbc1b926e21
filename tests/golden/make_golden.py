"""Generates the committed golden fixtures (tvl1 / refbuild need oracle/_ref, built by
`make -C oracle OPENCV_CONTRIB_DIR=<opencv_contrib source tree>`):
  farneback_*.npz  live CPU reference cv2.calcOpticalFlowFarneback (cv2 4.13.0 = opencv/opencv
                   modules/video/src/optflowgf.cpp, the function modules/optflow/src/interfaces.cpp:154-157 forwards to)
  tvl1_ref_*.npz   the reference's OWN CPU Dual TV-L1, opencv_contrib/modules/optflow/src/tvl1flow.cpp compiled
                   unmodified into oracle/_ref/libtvl1_ref.so (oracle/Makefile, oracle/ref_shim/)
  refbuild_*.npz   the same build on a second input (digest of the flow, to pin the C port bit for bit) and with an
                   initial flow (stride-8 sample); inputs are regenerated from oracle/synth.py and checked by digest
Brox and DensePyrLK need no fixture: their C models run at full size in the tests themselves
(tests/test_brox_fullsize_gpu.py, tests/test_denselk_fullsize_gpu.py).
python tests/golden/make_golden.py [farneback] [tvl1] [refbuild]   (no argument = farneback + tvl1)"""
import hashlib
import os
import sys

import numpy as np
import cv2

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import synth  # noqa: E402

CASES = {
    "box": (dict(), 1e-4, 0.02),
    "poly7": (dict(polyN=7, polySigma=1.5), 1e-4, 0.02),
    "gauss": (dict(flags=256), 2e-2, 0.2),
    "scale08": (dict(pyrScale=0.8, numLevels=3), 1e-4, 0.02),
}
WHAT = {a.split(":", 1)[0] for a in sys.argv[1:]} or {"farneback", "tvl1"}   # "tvl1:<case>" regenerates one TV-L1 case
for name, (kw, ncc_tol, epe_tol) in (CASES.items() if "farneback" in WHAT else ()):
    I0, I1, _ = synth.make_pair(144, 192, seed=11, kind="smooth")
    flow = cv2.calcOpticalFlowFarneback(I0, I1, None, kw.get("pyrScale", 0.5), kw.get("numLevels", 5), 13, 10,
                                        kw.get("polyN", 5), kw.get("polySigma", 1.1), kw.get("flags", 0))
    out = {"I0": I0, "I1": I1, "flow": flow.astype(np.float32), "ncc_tol": ncc_tol, "epe_tol": epe_tol,
           "cv2_version": cv2.__version__}
    out.update({"kw_" + k: v for k, v in kw.items()})
    np.savez_compressed(os.path.join(HERE, f"farneback_{name}.npz"), **out)
    print(name, flow.shape)

if "tvl1" in WHAT:
    from oracle import tvl1_cpu, tvl1_ref  # noqa: E402
    TV = {
        # the mapping the reference's GPU-vs-CPU test uses (cudaoptflow/test/test_optflow.cpp:456-460)
        "gpu_twin": dict(nscales=4, warps=5, epsilon=0.0, innerIterations=1, outerIterations=30, medianFiltering=1),
        "defaults": dict(),                                             # median 5, eps 0.01, 10 x 30
        "gamma": dict(gamma=0.5, medianFiltering=1, epsilon=0.0, innerIterations=5, outerIterations=4),
        "f32_median3": dict(medianFiltering=3, warps=2),
        # fixed work with the median filter on: what the engine's MEDIAN_FILTERING / MEDIAN_PERIOD knobs are checked against
        "median5_fixed": dict(nscales=3, warps=3, epsilon=0.0, innerIterations=10, outerIterations=3, medianFiltering=5),
    }
    only = {a.split(":", 1)[1] for a in sys.argv[1:] if a.startswith("tvl1:")}
    for name, kw in TV.items():
        if only and name not in only:
            continue
        I0, I1, gt = synth.make_pair(120, 160, seed=21, kind="affine", dtype="f32" if name.startswith("f32") else "u8")
        flow = tvl1_ref.calc(I0, I1, tvl1_cpu.TVL1Params(**kw))
        out = {"I0": I0, "I1": I1, "flow": flow, "gt": gt.astype(np.float32), "source": tvl1_ref.source()}
        out.update({"kw_" + k: v for k, v in kw.items()})
        np.savez_compressed(os.path.join(HERE, f"tvl1_ref_{name}.npz"), **out)
        print("tvl1", name, flow.shape, float(np.abs(flow).mean()))


if "refbuild" in WHAT:
    from oracle import tvl1_cpu, tvl1_ref  # noqa: E402
    sha1 = lambda a: hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()  # noqa: E731
    I0, I1, _ = synth.make_pair(150, 190, seed=9, kind="smooth")
    case = dict(h=150, w=190, seed=9, kind="smooth", sha1_I0=sha1(I0), sha1_I1=sha1(I1))
    kw = dict(warps=10, epsilon=0.0, innerIterations=1, outerIterations=30, medianFiltering=1)
    flow = tvl1_ref.calc(I0, I1, tvl1_cpu.TVL1Params(**kw))
    np.savez_compressed(os.path.join(HERE, "refbuild_port_check.npz"), flow_sha1=sha1(flow), **case,
                        **{"kw_" + k: v for k, v in kw.items()})
    kw = dict(nscales=1, warps=1, epsilon=0.0, innerIterations=1, outerIterations=2, medianFiltering=1,
              useInitialFlow=True)
    init = np.zeros(I0.shape + (2,), np.float32)
    init[..., 0] = 1.5
    flow = tvl1_ref.calc(I0, I1, tvl1_cpu.TVL1Params(**kw), init)
    assert abs(float(flow[..., 0].mean()) - 1.5) < 0.5, "the reference build ignored the initial flow"
    np.savez_compressed(os.path.join(HERE, "refbuild_initial_flow.npz"), flow_sha1=sha1(flow),
                        flow_s8=flow[::8, ::8].copy(), mean_u=float(flow[..., 0].mean(dtype=np.float64)), **case,
                        **{"kw_" + k: v for k, v in kw.items()})
    print("refbuild", flow.shape, float(flow[..., 0].mean()))
