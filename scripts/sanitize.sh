#!/bin/bash
# compute-sanitizer jobs for the hand-written kernels (SURVEY §5.2). Run on a GPU box:
#   gpurun -- 'bash scripts/sanitize.sh memcheck'      (or racecheck / synccheck / initcheck / all / late)
# The selection keeps the instrumented run short; the full suite is `pytest tests/test_gpu_kernels.py`.
#
# racecheck / synccheck target the kernels whose correctness rests on shared-memory hand-offs and barriers:
#   * wgmma GEMM family: TMA -> mbarrier -> wgmma -> accumulator + epilogue staging tiles (smem reuse across tiles)
#   * window_attn_fwd_tc: Q/K/V^T staging, P written back to smem between the two MMAs
#   * BN / CE / herding / triplet kernels: block reductions through shared memory
#   * fedcomm single-rank: the intra-block part of rank_barrier (__syncthreads_or around the flag spin)
# (the cross-rank flag protocol itself is system-scope global memory: racecheck does not model it; it is covered by
#  tests/dist_comm_check.py and scripts/comm_soak.py)
TOOL=${1:-memcheck}
SEL=${2:-"test_gemm_kmajor and 256-512-512 or test_conv_nhwc and 3-4-16-8 or test_lean_epilogue and 4096 or test_strided and 4-64-32-128 or test_fused_optimizer or test_fused_trained_l1_anchor or test_herding or test_fused_augmentation and default-dtype0 or test_comm_single_rank or test_window_attention_wgmma_forward and 37 or test_fused_triplet_loss and True-True or test_fused_kd_and_bce or test_batch_norm_shapes"}
mkdir -p gpurun_out
run() {
  local tool=$1
  timeout 1500 compute-sanitizer --tool "$tool" --error-exitcode 9 --log-file "gpurun_out/sanitizer_${tool}.log" \
    python -m pytest tests/test_gpu_kernels.py -q -x --timeout 1200 -p no:cacheprovider -k "$SEL" 2>&1 | tail -4
  echo "sanitizer ${tool} exit: $?"
  tail -5 "gpurun_out/sanitizer_${tool}.log"
}
# layer_ops.cu (compose / Swin token / dispatch-apply kernels): block reductions through shared memory + warp shuffles
run_late() {
  local tool=$1
  FLPR_LAYER_SELFCHECK=inprocess timeout 1500 compute-sanitizer --tool "$tool" --error-exitcode 9 \
    --log-file "gpurun_out/sanitizer_${tool}_layer_ops.log" \
    python -m pytest tests/test_zz_gpu_late.py -q -x --timeout 1200 -p no:cacheprovider \
      -k "compose_kernels or swin_token_kernels or apply_global_kernel or layer_norm_rows or window_merge_residual or gelu_act" 2>&1 | tail -4
  echo "sanitizer ${tool} (layer_ops) exit: $?"
  tail -5 "gpurun_out/sanitizer_${tool}_layer_ops.log"
}
if [ "$TOOL" = "late" ]; then
  for t in memcheck racecheck synccheck; do run_late $t; done
  exit 0
fi
if [ "$TOOL" = "all" ]; then
  for t in memcheck racecheck synccheck; do run $t; done
else
  run "$TOOL"
fi
