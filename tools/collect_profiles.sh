#!/bin/bash
# Turns what tools/profile_round.sh left in gpurun_out/ into the tracked summaries under profiles/ (run in the repo root).
set -e
R=${1:-r02}
O=gpurun_out
cp $O/r_bench.json profiles/${R}_bench.json
cp $O/r_vs_refcuda.txt profiles/${R}_vs_refcuda.txt
cp $O/r_lres_conv_table.txt profiles/${R}_lres_conv_table.txt
cp $O/r_convnd.txt profiles/${R}_convnd.txt
cat $O/r_tests.txt $O/r_smoke.txt > profiles/${R}_gpu_tests_and_smoke.txt
for w in lres sres; do
  python tools/summarize_launches.py $O/r_launches_$w.csv > profiles/${R}_launches_bench_$w.md
  gzip -c $O/r_launches_$w.csv > profiles/${R}_launches_bench_$w.csv.gz
done
for n in fl:filtered_lrelu_v3 wgrad:conv_wgrad_v2 igemm:conv_igemm adam:adam_step; do
  src=${n%%:*}; dst=${n##*:}
  [ -f $O/r_$src.ncu-rep ] && python tools/ncu_summary.py $O/r_$src.ncu-rep > profiles/${R}_ncu_$dst.md
done
cuobjdump -sass long-video-gan_b200/liblvg_ops.so | grep -oE "\b(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UBLKCP|SYNCS|FFMA|LDS\.128|STS\.128)\b[.A-Z0-9_]*" | sed 's/\..*//' | sort | uniq -c | sort -rn > profiles/${R}_sass_mnemonics.txt
ls -la profiles | tail -25
