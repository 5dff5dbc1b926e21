#!/bin/bash
# second GPU call of round 2: the whole GPU suite, smoke, the default bench line
mkdir -p gpurun_out
timeout 2400 python -m pytest tests -x -q -m gpu > gpurun_out/r2_pytest_all.log 2>&1
tail -15 gpurun_out/r2_pytest_all.log
timeout 600 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/r2_smoke.log 2>&1; tail -3 gpurun_out/r2_smoke.log
timeout 900 python bench.py --steps 5 --warmup 3 > gpurun_out/r2_bench_default.json 2> gpurun_out/r2_bench_default.err
tail -c 6000 gpurun_out/r2_bench_default.json; tail -5 gpurun_out/r2_bench_default.err
