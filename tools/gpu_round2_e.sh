#!/bin/bash
# fifth GPU call: Farneback occupancy variants, TV-L1 and Farneback tests
mkdir -p gpurun_out
timeout 300 python tools/gpu_probe_farn_r2.py 0 3 4 > gpurun_out/r2e_probe_farn.log 2>&1; cat gpurun_out/r2e_probe_farn.log
timeout 600 python -m pytest tests/test_tvl1_gpu.py tests/test_farneback_gpu.py -x -q -m gpu > gpurun_out/r2e_pytest.log 2>&1; tail -3 gpurun_out/r2e_pytest.log
