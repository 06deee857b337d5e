#!/bin/bash
# Race / memory checking of the hand-written kernels with compute-sanitizer on ONE GPU.
# The reference has no race detection at all (SURVEY §5); this is the device-side equivalent of a TSAN pass.
set -u
mkdir -p sanitizer_out
export PSB200_DEVICE_TIMEOUT=120
K="test_encode_gather_sgd and (identity or topk_f32 or scale_i8) and 3 and dtype0"
for tool in memcheck racecheck synccheck; do
  echo "=== compute-sanitizer --tool $tool"
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 --kernel-name kernel_substring=psb_ \
    python -m pytest tests/test_gpu_kernels.py -x -q -m gpu -k "$K or test_topk_wire_is_exact or test_adam_steps" \
    > sanitizer_out/sanitizer_$tool.log 2>&1
  echo "exit=$?"; grep -E "ERROR SUMMARY|passed|failed|RACECHECK SUMMARY|hazard" sanitizer_out/sanitizer_$tool.log | tail -4
done
# mode='sharded', two ranks on one GPU (spawned processes: compute-sanitizer follows them, --target-processes all), with and
# without the gated BcastLinear that acquires the counted PARAMS_READY
for tool in memcheck racecheck synccheck; do
  echo "=== compute-sanitizer --tool $tool (sharded, two ranks)"
  timeout 1800 compute-sanitizer --tool $tool --target-processes all --error-exitcode 9 --kernel-name kernel_substring=psb_ \
    python -m pytest tests/test_sharded_ps.py -x -q -m gpu -k "2-sgd-fp32 or bcast_linear" \
    > sanitizer_out/sanitizer_sharded_$tool.log 2>&1
  echo "exit=$?"; grep -E "ERROR SUMMARY|passed|failed|RACECHECK SUMMARY|hazard" sanitizer_out/sanitizer_sharded_$tool.log | tail -4
done
