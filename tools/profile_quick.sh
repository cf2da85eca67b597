#!/bin/bash
# The short version of tools/profile_round.sh for a tight GPU budget (ONE GPU, a few minutes): GPU tests,
# smoke, the bench line (reference-CUDA arm skipped: it does not change with this repo's kernels), the per-signature
# convolution table, two `ncu --set full` captures (weight gradient of a few-channel layer, forward kernel) and the launch
# list of the low-res bench command.   bash tools/profile_quick.sh   then   bash tools/collect_profiles.sh <round>
set -x
O=gpurun_out
mkdir -p $O
timeout 240 python -m pytest tests -m gpu -q 2>&1 | tail -4 | tee $O/r_tests.txt
timeout 120 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -14 | tee $O/r_smoke.txt
timeout 420 python bench.py --no-ref-cuda --cpu-budget 4 > $O/r_bench.json 2> $O/r_bench.err; tail -2 $O/r_bench.err; cut -c1-400 $O/r_bench.json
timeout 60 python tools/lres_conv_table.py > $O/r_lres_conv_table.txt 2>&1; tail -1 $O/r_lres_conv_table.txt
NCU="ncu --set full --clock-control none --import-source on -f"
timeout 120 $NCU -k regex:conv_wgrad_v2 -s 2 -c 1 -o $O/r_wgrad python tools/bench_convnd.py "lres D 32->64 1x3x3" > /dev/null 2>&1
timeout 120 $NCU -k regex:conv_igemm_kernel -s 2 -c 1 -o $O/r_igemm python tools/bench_convnd.py "lres G 512->512 3x3x3" > /dev/null 2>&1
timeout 200 ncu --metrics gpu__time_duration.sum --clock-control none -c 8000 --csv --log-file $O/r_launches_lres.csv python bench.py --steps 2 --warmup 3 --no-cpu --no-ref-cuda --workload lres > $O/r_launches_lres.log 2>&1
ls -la $O | tail -20
