#!/bin/bash
# programmatic dependent launch for the TV-L1 schedule: A/B against B2F_PDL=0 on one GPU
mkdir -p gpurun_out
for r in 1 2; do
  B2F_PDL=0 timeout 300 python tools/gpu_probe_r2.py 0:8:0 2>&1 | sed 's/^/pdl off  /'
  timeout 300 python tools/gpu_probe_r2.py 0:8:0 2>&1 | sed 's/^/pdl on   /'
done | tee gpurun_out/r2v_ab.log
