#!/usr/bin/env bash
# compute-sanitizer over the kernels whose correctness rests on hand-rolled mbarrier / cluster-barrier protocols
# (SURVEY.md §5; VERDICT r1 item 10).  memcheck on everything, racecheck (shared-memory hazards) on the same launches.
# Usage on the GPU box, from the repo root:  bash scripts/sanitize.sh [label]   -> gpurun_out/sanitize_<label>.log
set -u
label=${1:-r2}
out=gpurun_out/sanitize_$label.log
mkdir -p gpurun_out
CS=/usr/local/cuda/bin/compute-sanitizer
: > "$out"
for tool in memcheck racecheck; do
  for part in gemms attention llama ln_decoders encoders fusion fusion_mlp; do
    echo "==== $tool $part" | tee -a "$out"
    # --report-api-errors no: with it on, memcheck's one and only report is the CUDA runtime's own lazy-loading probe
    # (cuKernelGetFunction -> CUDA_ERROR_INVALID_HANDLE inside the first cudaLaunchKernel of the process, handled by the
    # runtime; profiles/r2_sanitizer.log keeps that run too) -- not a memory error of a kernel
    timeout 900 $CS --tool $tool --report-api-errors no --print-limit 20 --error-exitcode 9 python scripts/sanitize_driver.py $part > gpurun_out/sanitize_last.log 2>&1
    rc=$?
    grep -E "ERROR SUMMARY|RACECHECK SUMMARY|ok$|Error|error:|hazard" gpurun_out/sanitize_last.log | head -20 | tee -a "$out"
    grep -B2 -A14 -E "Invalid|Misaligned|out of bounds|uninitialized" gpurun_out/sanitize_last.log | head -60 >> "$out"
    echo "exit $rc" | tee -a "$out"
  done
done
