#!/bin/bash
# on the GPU box: capture a few kernels with ncu --set full and keep only the raw-metric CSV (the .ncu-rep files are too big to bring back)
set -u
mkdir -p gpurun_out
cap() {  # name, kernel regex, skip, count, command...
  local name=$1 rx=$2 skip=$3 cnt=$4; shift 4
  timeout 280 ncu --set full --clock-control none -k regex:"$rx" -s $skip -c $cnt -o /tmp/$name "$@" > /dev/null 2>&1
  ncu -i /tmp/$name.ncu-rep --page raw --csv > gpurun_out/ncu_$name.csv 2>/dev/null
  rm -f /tmp/$name.ncu-rep
  wc -c gpurun_out/ncu_$name.csv
}
cap snac 'ru_fused|conv_gemm|final_nlc|dw7' 37 37 python tools/profile_snac.py 8 1024
cap whisper 'mha_tc|mel_log|tc_gemm_kernel<128>|layernorm' 30 12 python tools/profile_whisper.py 16 2
cap step 'tc_gemm|add_rmsnorm|attn_decode' 210 8 python tools/profile_step.py 320 3
