"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol
include/b200flow.h declares, and its host-only entry points behave (no compute without a GPU)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    from opencv_contrib_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        g.build()
    return _lib.lib()


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200flow.h")).read()
    return sorted(set(re.findall(r"B2F_API\s+[\w\s\*]+?\b(b2f_\w+)\s*\(", src)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    from opencv_contrib_b200 import _lib
    decl = declared_symbols()
    assert len(decl) >= 20
    bound = {n for n, _, _ in _lib.SYMBOLS}
    for name in decl:
        assert hasattr(lib, name), f"{name} declared in b200flow.h but not exported"
        assert name in bound, f"{name} not bound in _lib.SYMBOLS"


def test_defaults_match_reference_create(lib):
    from opencv_contrib_b200 import _lib
    p = _lib.b2f_tvl1_params()
    lib.b2f_tvl1_default_params(C.byref(p))
    # cudaoptflow.hpp:375-385
    assert (p.tau, p.lambda_, p.theta, p.nscales, p.warps, p.epsilon, p.iterations, p.scale_step, p.gamma,
            p.use_initial_flow) == (0.25, 0.15, 0.3, 5, 5, 0.01, 300, 0.8, 0.0, 0)
    f = _lib.b2f_farneback_params()
    lib.b2f_farneback_default_params(C.byref(f))
    # cudaoptflow.hpp:285-293
    assert (f.num_levels, f.pyr_scale, f.fast_pyramids, f.win_size, f.num_iters, f.poly_n, f.poly_sigma,
            f.flags) == (5, 0.5, 0, 13, 10, 5, 1.1, 0)
    b = _lib.b2f_brox_params()
    lib.b2f_brox_default_params(C.byref(b))
    assert (b.alpha, b.gamma, b.scale_factor, b.inner_iterations, b.outer_iterations, b.solver_iterations) == (
        0.197, 50.0, 0.8, 5, 150, 10)  # cudaoptflow.hpp:179-185
    d = _lib.b2f_denselk_params()
    lib.b2f_denselk_default_params(C.byref(d))
    assert (d.win_width, d.win_height, d.max_level, d.iters, d.use_initial_flow) == (13, 13, 3, 30, 0)


def test_python_mirror_getters_setters_and_names(lib):
    import opencv_contrib_b200 as ocb
    a = ocb.OpticalFlowDual_TVL1_create()
    assert a.getDefaultName() == "DenseOpticalFlow.OpticalFlowDual_TVL1"  # tvl1flow.cpp:122
    assert a.getNumIterations() == 300 and a.getNumWarps() == 5 and a.getScaleStep() == 0.8
    a.setNumIterations(30); a.setNumWarps(10); a.setEpsilon(0.0); a.setGamma(0.5); a.setUseInitialFlow(True)
    assert (a.getNumIterations(), a.getNumWarps(), a.getEpsilon(), a.getGamma(), a.getUseInitialFlow()) == (
        30, 10, 0.0, 0.5, True)
    f = ocb.FarnebackOpticalFlow_create()
    assert f.getDefaultName() == "DenseOpticalFlow.FarnebackOpticalFlow"  # farneback.cpp:132
    f.setWinSize(15); f.setFlags(ocb.OPTFLOW_FARNEBACK_GAUSSIAN)
    assert f.getWinSize() == 15 and f.getFlags() == 256 and f.getPolyN() == 5


def test_null_and_bad_arguments_fail_loudly(lib):
    from opencv_contrib_b200 import _lib
    h = C.c_void_p()
    assert lib.b2f_tvl1_create(None, C.byref(h)) == 0 and h.value
    img = _lib.b2f_image(None, 0, 0, 0, 0)
    assert lib.b2f_calc(h, None, None, None, None) == 1           # B2F_BAD_ARG
    assert lib.b2f_calc(h, C.byref(img), C.byref(img), C.byref(img), None) == 1
    assert lib.b2f_set_param(h, 12345, 1.0) == 1
    v = C.c_double(-1.0)
    active = _lib.PARAM["engine"]["active_path"]
    assert lib.b2f_get_param(h, active, C.byref(v)) == 1 and v.value == -1.0  # no calc yet: no level to report
    assert lib.b2f_set_param(h, active, 1.0) == 1                               # read-only
    assert b"B2F_BAD_ARG" in lib.b2f_status_string(1)
    lib.b2f_destroy(h)
    assert lib.b2f_tvl1_create(None, None) == 1


def test_active_path_ids_match_header():
    from opencv_contrib_b200 import _lib
    src = open(os.path.join(ROOT, "include", "b200flow.h")).read()
    flags = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r"B2F_TVL1_PATH_(\w+)\s*=\s*(\d+)", src)}
    assert flags == _lib.TVL1_PATH
    farn = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r"B2F_FARN_PATH_(\w+)\s*=\s*(\d+)", src)}
    assert farn == _lib.FARN_PATH
    assert len(set(farn.values())) == len(farn) and 0 not in farn.values()  # 0 means "no iteration ran"
    brox = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r"B2F_BROX_PATH_(\w+)\s*=\s*(\d+)", src)}
    assert brox == _lib.BROX_PATH
    assert len(set(brox.values())) == len(brox) and 0 not in brox.values() and max(brox.values()) < 256  # bits 0-7
    assert int(re.search(r"B2F_ENGINE_ACTIVE_PATH\s*=\s*(\d+)", src).group(1)) == _lib.PARAM["engine"]["active_path"]


def test_header_is_plain_c99(tmp_path):
    """include/b200flow.h is the drop-in boundary: it must compile as C (no C++ types, no torch types)."""
    import shutil
    import subprocess
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if not gcc:
        pytest.skip("no C compiler")
    src = tmp_path / "abi.c"
    src.write_text('#include "b200flow.h"\n'
                   "int main(void) { b2f_error_stats s; b2f_sparselk_params p; b2f_image im; (void)s; (void)p; (void)im;\n"
                   "  return B2F_OK; }\n")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only",
                        "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_cpp_adapter_real_opencv_branch_compiles(tmp_path):
    """include/b200flow/cudaoptflow_compat.hpp selects its real-OpenCV branch whenever OpenCV's core headers are on
    the include path; the image has none, so that branch is compiled here (syntax only) against declaration-only
    stand-ins that keep opencv core's signatures (getGpuMat() by value, getGpuMatRef() by reference, cv::noArray())."""
    import shutil
    import subprocess
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    cuda_inc = "/usr/local/cuda/include"
    if not gxx or not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("no C++ compiler / CUDA headers")
    cpp = os.path.join(ROOT, "tests", "cpp")
    r = subprocess.run([gxx, "-std=c++17", "-fsyntax-only", "-DB200FLOW_WITH_OPENCV", "-I", os.path.join(cpp, "opencv_stub"),
                        "-I", os.path.join(ROOT, "include"), "-I", cuda_inc, os.path.join(cpp, "opencv_branch_syntax.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
