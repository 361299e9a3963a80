#!/bin/bash
# bench + ncu evidence, one GPU.  Small summaries under gpurun_out/ (reports stay on the box).
mkdir -p gpurun_out /tmp/prof
TAG=${1:-r01}
timeout 900 python bench.py --gpus 1 > gpurun_out/bench_$TAG.json 2> gpurun_out/bench_$TAG.err
echo "bench exit $?"; tail -c 2500 gpurun_out/bench_$TAG.json
timeout 600 python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/ref_$TAG.json 2>> gpurun_out/bench_$TAG.err
tail -c 300 gpurun_out/ref_$TAG.json
# launch list of the bench command (cold-cache, serialised: compare shares)
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 4000 --csv \
    --log-file gpurun_out/launches_$TAG.csv python bench.py --steps 1 --warmup 3 --no-cpu > gpurun_out/ncu_bench_$TAG.log 2>&1
echo "ncu launches exit $?"; wc -l gpurun_out/launches_$TAG.csv
cap() {  # name regex skip count
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:"$2" -s $3 -c $4 \
      -o /tmp/prof/$1 -f python tools/one_build.py > gpurun_out/ncu_$1_$TAG.log 2>&1
  ncu -i /tmp/prof/$1.ncu-rep --page raw --csv > gpurun_out/raw_$1_$TAG.csv 2>/dev/null
  ls -la /tmp/prof/$1.ncu-rep
}
cap induce 'k_induce' 4 4
cap ospass 'k_os_pass' 12 3
cap stream 'k_cls_block_state|k_pack|k_name_flags|k_lcp_direct|k_unrename' 7 7
cap scans 'k_scan_apply|k_scan_reduce|k_os_hist|k_multi_key_list' 20 8
du -sh gpurun_out
