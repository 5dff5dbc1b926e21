#!/bin/bash
# third GPU call of round 2: new build (31-op TV-L1 math, device-side epsilon loop, Farneback running sums):
# conditional-graph sanity, TV-L1 + Farneback test files, probes, ncu captures of the top kernels
mkdir -p gpurun_out
timeout 60 tools/ubench/cond_graph_test > gpurun_out/r2_cond_graph.log 2>&1; cat gpurun_out/r2_cond_graph.log
timeout 1500 python -m pytest tests/test_tvl1_gpu.py tests/test_farneback_gpu.py tests/test_adjacent_gpu.py -x -q -m gpu > gpurun_out/r2c_pytest.log 2>&1
tail -8 gpurun_out/r2c_pytest.log
timeout 300 python tools/gpu_probe_farneback.py 2>&1 | tail -12 > gpurun_out/r2c_probe_farn.log; cat gpurun_out/r2c_probe_farn.log
python - <<'PY' > gpurun_out/r2c_cluster_info.log 2>&1
import ctypes as C, sys, os
sys.path.insert(0, os.getcwd())
import torch
torch.zeros(1, device="cuda")
from opencv_contrib_b200 import _lib
PY
bash tools/ncu_capture_r2.sh > gpurun_out/r2c_ncu.log 2>&1; tail -6 gpurun_out/r2c_ncu.log
