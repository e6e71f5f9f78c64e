#!/bin/bash
# compute-sanitizer passes over the small-shape GPU tests (development tool, run under gpurun).
# memcheck: out-of-bounds / misaligned accesses; racecheck: shared-memory hazards; synccheck: barrier misuse.
#   bash tools/sanitize.sh [tools...]      default: memcheck synccheck (racecheck takes ~5x longer)
set -u
OUT=gpurun_out
mkdir -p $OUT
TOOLS=${@:-memcheck synccheck}
SEL='rmsnorm or embed or rope or kv_append or hyena_operator or hyena_step or continuation or (gemm_all and 300-512) or (attention_vs_oracle and 300) or decode_attention or stateful'
SEL="$SEL or (rotary_epilogue and 129) or peer_scattered or sampler_greedy or (sampler_distribution and 50) or device_loop_equals or tokenise or (fused_unembed and 129)"
FILES="tests/test_gpu_parity.py tests/test_gpu_generation.py tests/test_gpu_frontend.py tests/test_gpu_fullsize.py"
for tool in $TOOLS; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 7 --print-limit 20 python -m pytest $FILES -q -x -m gpu -k "$SEL" > $OUT/sanitizer_$tool.log 2>&1
  echo "$tool rc=$? $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' $OUT/sanitizer_$tool.log | tr '\n' ' ')"
done
