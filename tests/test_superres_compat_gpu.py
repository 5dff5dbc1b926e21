"""The C++ super-resolution adapter (include/b200flow/superres_compat.hpp) used from a C++ call site
(tests/cpp/test_superres_compat.cpp) gives the same 8-bit frames as the Python path (same library, same kernels)."""
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_superres_compat")


@pytest.mark.parametrize("flow,cn", [("zero", 3), ("farneback", 1), ("brox", 4)])
def test_cpp_call_site_matches_python_path(cuda_device, tmp_path, flow, cn):
    import torch
    import opencv_contrib_b200 as ocb
    rows, cols, n = 20, 24, 4
    rng = np.random.default_rng(cn)
    frames = [rng.integers(0, 256, (rows, cols, cn), dtype=np.uint8) for _ in range(n)]
    pin, pout = tmp_path / "in.raw", tmp_path / "out.raw"
    np.stack(frames).tofile(pin)
    r = subprocess.run([EXE, flow, str(rows), str(cols), str(cn), str(n), str(pin), str(pout)], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    orows, ocols = rows * 2 - 14, cols * 2 - 14
    got = np.fromfile(pout, np.uint8).reshape(n, orows, ocols, cn)

    class Zero:
        def calc(self, f0, f1, u, v):
            return u, v  # zero-filled by the caller

    s = ocb.createSuperResolution_BTVL1_CUDA()
    s.setScale(2), s.setIterations(5), s.setTemporalAreaRadius(1), s.setLambda(0.05)
    if flow == "zero":
        s.setOpticalFlow(Zero())
    elif flow == "brox":
        b = ocb.createOptFlow_Brox_CUDA()
        b.setOuterIterations(4)
        s.setOpticalFlow(b)
    s.setInput([f if cn > 1 else f[..., 0] for f in frames])
    want = []
    while (o := s.nextFrame()) is not None:
        want.append(o.cpu().numpy().reshape(orows, ocols, cn))
    assert len(want) == n
    assert np.array_equal(got, np.stack(want))
