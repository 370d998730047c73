#!/bin/sh
# compute-sanitizer over the kernels added late in round 2: the STATS epilogue of conv_tc_kernel (32/64-column chunks, 8 epilogue
# warps, CTA pair), partial_reduce_kernel, pack_gather1_kernel (logs -> $OUT, default /tmp/rsb_sanitize).
SAN=/usr/local/cuda/bin/compute-sanitizer
SEL='test_conv_stats_epilogue_partials_fold_to_float64_batchnorm or test_relu_maxpool_final_pack_unpack_kernels'
OUT=${OUT:-/tmp/rsb_sanitize}
mkdir -p "$OUT"
for TOOL in memcheck synccheck; do
  timeout 420 $SAN --tool $TOOL --log-file $OUT/sanitizer_r2b_$TOOL.log python -m pytest tests/test_conv_gpu.py tests/test_train_gpu.py -m gpu -q -x -k "$SEL" > $OUT/sanitizer_r2b_${TOOL}_pytest.log 2>&1
  echo "== $TOOL: pytest rc $? ; $(tail -1 $OUT/sanitizer_r2b_${TOOL}_pytest.log)"
  grep -E "ERROR SUMMARY|Error|hazard" $OUT/sanitizer_r2b_$TOOL.log | sort | uniq -c | head -8
done
