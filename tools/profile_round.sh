#!/bin/bash
# Runs on the GPU: tests, bench, ncu launch list, one full ncu capture per hot kernel.
# tools/summarize_profiles.py turns the raw outputs into summaries under profiles/ (not tracked by git).
set -u
O=gpurun_out
mkdir -p $O
cp incubator_pegasus_b200/libpegasus_b200.so $O/lib_at_profile.so
timeout 900 python -m pytest tests -x -q -m gpu > $O/final_tests.log 2>&1; tail -2 $O/final_tests.log
timeout 1500 python bench.py --steps 5 --warmup 3 > $O/final_bench.json 2> $O/final_bench.err; head -c 300 $O/final_bench.json; echo
B="python bench.py --skip-cpu --skip-e2e --skip-sharded --skip-sweep --skip-ycsb"
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file $O/final_launches.csv $B --steps 2 --warmup 1 > $O/final_launches.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:k_walk -s 1 -c 1 -f -o $O/final_k_walk $B --steps 2 --warmup 1 --skip-reads > $O/final_ncu_walk.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:k_emit -s 1 -c 1 -f -o $O/final_k_emit $B --steps 2 --warmup 1 --skip-reads > $O/final_ncu_emit.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:k_get -s 1 -c 1 -f -o $O/final_k_get $B --steps 1 --warmup 1 > $O/final_ncu_get.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:k_scan_fwd -s 1 -c 1 -f -o $O/final_k_scan_fwd $B --steps 1 --warmup 1 > $O/final_ncu_scan.log 2>&1
ls -la $O | grep final
