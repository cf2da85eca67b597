#!/bin/bash
# Regenerates the evidence on an H100 (one GPU): GPU tests, smoke, the bench line,
# ncu launch lists of the bench commands, `ncu --set full` captures of the hot kernels, per-op tables.
#   bash tools/profile_round.sh   then   bash tools/collect_profiles.sh <round>
set -x
O=gpurun_out
python -m pytest tests -m gpu -q 2>&1 | tail -3 | tee $O/r_tests.txt
python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -14 | tee $O/r_smoke.txt
python bench.py > $O/r_bench.json 2> $O/r_bench.err; tail -2 $O/r_bench.err; cut -c1-300 $O/r_bench.json
python tools/bench_vs_refcuda.py > $O/r_vs_refcuda.txt 2>&1
python tools/lres_conv_table.py > $O/r_lres_conv_table.txt 2>&1
python tools/bench_convnd.py > $O/r_convnd.txt 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 8000 --csv --log-file $O/r_launches_lres.csv python bench.py --steps 2 --warmup 3 --no-cpu --no-ref-cuda --workload lres > $O/r_launches_lres.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 8000 --csv --log-file $O/r_launches_sres.csv python bench.py --steps 1 --warmup 3 --no-cpu --no-ref-cuda --workload sres > $O/r_launches_sres.log 2>&1
NCU="ncu --set full --clock-control none --import-source on -f"
$NCU -k regex:filtered_lrelu_v3 -c 4 -o $O/r_fl python tools/fl_probe.py 1 > /dev/null 2>&1
$NCU -k regex:conv_wgrad_v2 -s 2 -c 1 -o $O/r_wgrad python tools/bench_convnd.py "lres G 512->512 3x3x3" > /dev/null 2>&1
$NCU -k regex:conv_igemm_kernel -s 2 -c 1 -o $O/r_igemm python tools/bench_convnd.py "lres G 512->512 3x3x3" > /dev/null 2>&1
$NCU -k regex:adam_step -c 1 -o $O/r_adam python -m pytest tests/test_flat_optim.py -m gpu -q -k sanitises > /dev/null 2>&1
ls -la $O | tail -30
