#!/bin/bash
# sixth GPU call: new defaults (separable warp @40 regs, Farneback iteration @80 regs): full suite, smoke, probes,
# default bench line, final ncu captures and the launch list of the bench command
mkdir -p gpurun_out
timeout 2400 python -m pytest tests -x -q -m gpu > gpurun_out/r2f_pytest_all.log 2>&1; tail -6 gpurun_out/r2f_pytest_all.log
timeout 600 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/r2f_smoke.log 2>&1; tail -2 gpurun_out/r2f_smoke.log
timeout 300 python tools/gpu_probe_farn_r2.py 0 2 4 > gpurun_out/r2f_probe_farn.log 2>&1; cat gpurun_out/r2f_probe_farn.log
timeout 900 python bench.py --steps 5 --warmup 3 > gpurun_out/r2f_bench_default.json 2> gpurun_out/r2f_bench_default.err
tail -c 800 gpurun_out/r2f_bench_default.json; tail -3 gpurun_out/r2f_bench_default.err
NCU="ncu --set full --clock-control none --import-source on --launch-count 1 -f"
timeout 300 $NCU --kernel-name regex:k_tvl1_blocked_tma --launch-skip 165 -o gpurun_out/prof_tvl1_tma_r2f python tools/prof_one.py tvl1 8 1 0 > /dev/null 2>&1
timeout 300 $NCU --kernel-name regex:k_tvl1_warp_sep --launch-skip 45 -o gpurun_out/prof_tvl1_warp_r2f python tools/prof_one.py tvl1 8 1 0 > /dev/null 2>&1
timeout 300 $NCU --kernel-name regex:k_farn_iter_fast --launch-skip 55 -o gpurun_out/prof_farn_iter_r2f python tools/prof_one.py farneback 0 1 > /dev/null 2>&1
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 1400 --csv --log-file gpurun_out/launches_r2_tvl1.csv python bench.py --steps 1 --warmup 3 --pairs 2 --streams 1 --no-cpu --no-extras --workload tvl1 > gpurun_out/r2f_bench_under_ncu.log 2>&1
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 900 --csv --log-file gpurun_out/launches_r2_farn.csv python bench.py --steps 1 --warmup 3 --pairs 2 --streams 1 --no-cpu --no-extras --workload farneback > gpurun_out/r2f_bench_under_ncu_farn.log 2>&1
ls -la gpurun_out/*r2f* gpurun_out/launches_r2_*
