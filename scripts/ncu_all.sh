#!/bin/bash
# ncu --set full captures of one launch (or a few) per kernel family -> gpurun_out/prof_*.ncu-rep (read on the CPU box
# with scripts/ncu_summary.py). Run under gpurun on ONE GPU.
set -u
mkdir -p gpurun_out
N="ncu --set full --clock-control none --import-source on"
run() { # name, what, regex, skip, count
  timeout 240 $N -k "regex:$3" -s "$4" -c "$5" -f -o "gpurun_out/prof_$1" python scripts/ncu_targets.py "$2" > "gpurun_out/prof_$1.log" 2>&1
  echo "$1 rc=$? $(ls -la gpurun_out/prof_$1.ncu-rep 2>/dev/null | awk '{print $5}')"
}
run head_gemm   head  "gemm_bf16_wgmma"        120 14
run head_opt    head  "fused_opt"                4   2
run head_bn     head  "bn_(affine_rows|bwd_reduce|bwd_rows|finalize|fold)" 110 10
run head_ce     head  "ce_ls|gap_"               6   3
run trunk_conv  trunk "gemm_bf16_wgmma|maxpool|s2d" 60 12
run swin_attn   swin  "window_attn_fwd_tc"       12  3
run comm        comm  "fed_"                     2   3
run misc        misc  "triplet_mine|herding|rank_eval|augment" 0 8
