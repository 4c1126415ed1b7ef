#!/bin/bash
# ncu captures of one cfg3_train step (run on a GPU machine: bash tools/ncu_capture_train_step.sh).  Numbers printed by bench.py
# under ncu are never bench values; the .ncu-rep files stay in $T and only their summaries go to results/.
mkdir -p results
T=/tmp/ncu_r2
mkdir -p $T
ncu --set full --clock-control none --import-source on -k regex:'attention|layernorm|conv_head_final|adamw|sumsq|colsum16|attn_delta' -s 135 -c 45 -f -o $T/rows python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-extras > results/r2f_ncu_rows.log 2>&1
python tools/ncu_summary.py $T/rows.ncu-rep results/r2f_rowkernels_ncu_full_summary.csv >> results/r2f_ncu_rows.log 2>&1
ncu -i $T/rows.ncu-rep --page source --csv -k regex:attention_bwd > results/r2f_attention_bwd_source.csv 2>/dev/null
ncu -i $T/rows.ncu-rep --page source --csv -k regex:layernorm_bwd_vec > results/r2f_layernorm_bwd_source.csv 2>/dev/null
ls -la $T >> results/r2f_ncu_rows.log
rm -f $T/rows.ncu-rep
ncu --set full --clock-control none -k regex:gemm_wgmma -s 174 -c 58 -f -o $T/gemm python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-extras > results/r2f_ncu_gemm.log 2>&1
python tools/ncu_summary.py $T/gemm.ncu-rep results/r2f_gemm_ncu_full_summary.csv >> results/r2f_ncu_gemm.log 2>&1
rm -f $T/gemm.ncu-rep
ncu --metrics gpu__time_duration.sum --clock-control none -s 600 -c 400 --csv --log-file results/r2f_launches_cfg3_train.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-extras > results/r2f_ncu_launches.log 2>&1
du -sh results >> results/r2f_ncu_rows.log
