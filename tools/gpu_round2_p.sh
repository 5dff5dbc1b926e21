#!/bin/bash
# sixteenth GPU call: TMA loads / stores issued by ten / six warps instead of one lane: clocks, timing
mkdir -p gpurun_out
timeout 300 python tools/gpu_probe_tile_clocks.py 2>&1 | grep -E "iters 8" > gpurun_out/r2p_clocks.log; cat gpurun_out/r2p_clocks.log
timeout 300 python tools/gpu_probe_r2.py 0:8:3 > gpurun_out/r2p_probe.log 2>&1; cat gpurun_out/r2p_probe.log
