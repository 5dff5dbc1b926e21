#!/bin/bash
# fourth GPU call: 3-MUFU math restored: TV-L1 tests, default bench line
mkdir -p gpurun_out
timeout 900 python -m pytest tests/test_tvl1_gpu.py -x -q -m gpu > gpurun_out/r2d_pytest.log 2>&1; tail -4 gpurun_out/r2d_pytest.log
timeout 900 python bench.py --steps 5 --warmup 3 > gpurun_out/r2d_bench_default.json 2> gpurun_out/r2d_bench_default.err
tail -c 1500 gpurun_out/r2d_bench_default.json; tail -5 gpurun_out/r2d_bench_default.err
