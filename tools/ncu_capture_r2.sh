# round-2 ncu captures (one GPU; each capture replays ONE launch ~40 times): .ncu-rep files land in gpurun_out/
set -x
cd $GRAFT_REPO_ROOT
NCU="ncu --set full --clock-control none --import-source on --launch-count 1 -f"
# TV-L1 scalar persistent TMA kernel, level 0, K = 8 (200 iteration launches per calc, level 0 = the last 40)
timeout 300 $NCU --kernel-name regex:k_tvl1_blocked_tma --launch-skip 165 -o gpurun_out/prof_tvl1_tma_r2a python tools/prof_one.py tvl1 8 1 0 > /dev/null 2>&1
# Farneback fused iteration, level 0 (60 iteration launches per calc, level 0 = the last 10)
timeout 300 $NCU --kernel-name regex:k_farn_iter_fast --launch-skip 55 -o gpurun_out/prof_farn_iter_r2a python tools/prof_one.py farneback 0 1 > /dev/null 2>&1
ls -la gpurun_out/*r2a.ncu-rep
