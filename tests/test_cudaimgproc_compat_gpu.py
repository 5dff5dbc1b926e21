"""The C++ corner adapter (include/b200flow/cudaimgproc_compat.hpp) used from a C++ call site
(tests/cpp/test_cudaimgproc_compat.cpp) gives the response and the corners of oracle/corners_model.py bit for bit, and
a released output for an image without candidates."""
import os
import subprocess

import numpy as np
import pytest

from oracle import corners_model as M
from oracle import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_cudaimgproc_compat")


@pytest.mark.parametrize("shape", [(240, 320), (33, 65)])
def test_cpp_call_site_matches_model(cuda_device, tmp_path, shape):
    rows, cols = shape
    img = np.clip(np.rint(synth.texture(rows, cols, 31)), 0, 255).astype(np.uint8)
    pin, peig, pc = tmp_path / "in.raw", tmp_path / "eig.raw", tmp_path / "c.raw"
    img.tofile(pin)
    r = subprocess.run([EXE, str(rows), str(cols), str(pin), str(peig), str(pc)], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    eig = np.fromfile(peig, np.float32).reshape(rows, cols)
    assert np.array_equal(eig, M.response(img, 5, 5, M.BORDER_REFLECT, True, 0.04))
    raw = np.fromfile(pc, np.float32)
    n = int(raw[:1].view(np.int32)[0])
    want, _ = M.gftt(img, 500, 0.01, 3.0)
    assert n == len(want) > 0 and np.array_equal(raw[1:].reshape(-1, 2), want)
