#!/bin/bash
# alternating tile walking direction of the iteration passes (first region of a pass = data the previous kernel touched last): A/B on one box
mkdir -p gpurun_out
for r in 1 2; do
  B2F_DBG_TVL1_NOREV=1 timeout 300 python tools/gpu_probe_r2.py 0:8:0 2>&1 | sed 's/^/forward      /'
  timeout 300 python tools/gpu_probe_r2.py 0:8:0 2>&1 | sed 's/^/alternating  /'
done | tee gpurun_out/r2w_ab.log
