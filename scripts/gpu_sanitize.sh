#!/bin/sh
# compute-sanitizer over one small convolution per kernel variant (fast, strict 3-MMA pair, strict N-concatenated, K-chunked) and
# one weight-gradient case. The logs go to $OUT/sanitizer_*.log (default /tmp/rsb_sanitize).
SAN=/usr/local/cuda/bin/compute-sanitizer
SEL='test_conv_case_matches_cpu_reference[3] or test_conv_cta_pair_matches_single_cta[1] or test_split_conv_case_matches_fp64_reference[0] or test_split_conv_case_matches_fp64_reference[5] or test_split_conv_case_matches_fp64_reference[15] or test_wgrad_split_k_scratch_matches_cpu_emulation[2]'
OUT=${OUT:-/tmp/rsb_sanitize}
mkdir -p "$OUT"
for TOOL in memcheck synccheck racecheck; do
  timeout 420 $SAN --tool $TOOL --log-file $OUT/sanitizer_$TOOL.log python -m pytest tests/test_conv_gpu.py tests/test_train_gpu.py -m gpu -q -x -k "$SEL" > $OUT/sanitizer_${TOOL}_pytest.log 2>&1
  echo "== $TOOL: pytest rc $? ; $(tail -1 $OUT/sanitizer_${TOOL}_pytest.log)"
  grep -E "ERROR SUMMARY|RACECHECK SUMMARY|Error|hazard" $OUT/sanitizer_$TOOL.log | sort | uniq -c | head -8
done
