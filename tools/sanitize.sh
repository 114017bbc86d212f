#!/bin/bash
# compute-sanitizer over the small-size GPU parity tests (memcheck, then racecheck + synccheck on the kernels that use
# shared memory).  Slow (10-100x): only the tests whose sizes are small.   bash tools/sanitize.sh [log-dir]
set -u
out=${1:-sanitizer_out}
mkdir -p "$out"
SMALL='test_field_arithmetic or test_point_arithmetic or test_bucket_reduction_kernels or (test_ntt_matches_oracle and not 16) or test_multiexp_g1_matches_oracle or test_multiexp_g2_matches_oracle or test_affine_rounds or test_multiexp_error_semantics or test_prove_mimc322 or test_fr_dot'
for tool in memcheck racecheck synccheck; do
    timeout 1200 compute-sanitizer --tool $tool --error-exitcode 9 --launch-timeout 120 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "$SMALL" > "$out/sanitizer_$tool.log" 2>&1
    echo "$tool rc=$?"; grep -E "ERROR SUMMARY|passed|failed|RACECHECK SUMMARY|Error" "$out/sanitizer_$tool.log" | tail -5
done
# proving from the witness on a sharded key: the owner stage and the begin / end pair at small sizes
timeout 1200 compute-sanitizer --tool memcheck --error-exitcode 9 --launch-timeout 120 python -m pytest tests/test_gpu_r1cs_shard.py -x -q -m gpu \
    -k "test_owner_mimc322 or test_owner_from_assembly or test_errors" > "$out/sanitizer_memcheck_r1cs_shard.log" 2>&1
echo "memcheck r1cs_shard rc=$?"; grep -E "ERROR SUMMARY|passed|failed|Error" "$out/sanitizer_memcheck_r1cs_shard.log" | tail -5
