#!/bin/bash
# compute-sanitizer over the kernel tests (1 GPU): memcheck, racecheck (shared-memory hazards of
# the TMA pipelines), synccheck.  Each tool under its own limit; output -> gpurun_out/sanitizer.txt
mkdir -p gpurun_out
OUT=gpurun_out/sanitizer.txt
echo "# compute-sanitizer on tests/test_gpu_kernels.py + the doorbell / fused-fp8 store tests (1 GPU)" > $OUT
run() {
    local tool=$1 secs=$2; shift 2
    echo "== $tool" >> $OUT
    timeout -k 10 $secs compute-sanitizer --tool $tool --target-processes all "$@" 2>&1 \
        | grep -v "^$" | grep "COMPUTE-SANITIZER\|passed\|failed\|SUMMARY\|hazard\|Invalid\|Error\|error" | head -40 >> $OUT
    local rc=${PIPESTATUS[0]}
    echo "rc=$rc" >> $OUT
    echo "== $tool rc=$rc"; tail -4 $OUT
    if [ $rc -eq 124 ] || [ $rc -eq 137 ]; then echo "ABORT: $tool ran into its limit"; exit 1; fi
}
K="python -m pytest tests/test_gpu_kernels.py -q -x -p no:cacheprovider"
run memcheck 420 $K
run memcheck 300 python -m pytest tests/test_gpu_store.py tests/test_gpu_features.py -q -x -p no:cacheprovider -k "doorbell_worker_serves or fp8_fused or unbalanced"
run racecheck 420 $K -k "pipeline or cluster or fan or fp8 or swizzle"
run synccheck 300 $K
