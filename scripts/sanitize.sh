#!/bin/bash
# Race / memory checks for the sm_90a kernels (run on a GPU box; SURVEY 5.2).  compute-sanitizer does not
# see cross-device races: those are covered by tests/test_gpu_v2.py (replicas must stay bit-identical, protocol
# fuzz with randomized delays) and by the step-stamped flag protocol (flags are never reset, only compared).
#
#   scripts/sanitize.sh [memcheck|synccheck|racecheck ...]      default: memcheck synccheck
#
# Notes from earlier runs:
#  * racecheck does NOT finish within 15 min on the v2 kernels (every shared-memory access is tracked): run it on a
#    single test (-k gram) with its own timeout, never inside a budgeted 8-GPU call;
#  * the CUDA-graph capture test is excluded: cudaStreamBeginCapture makes the sanitizer report API errors
#    (cudaErrorStreamCaptureUnsupported) for its own instrumentation calls, which are not kernel bugs.
set -e
tools=${@:-memcheck synccheck}
mkdir -p gpurun_out
for tool in $tools; do
  echo "== compute-sanitizer --tool $tool"
  limit=600; [ "$tool" = racecheck ] && limit=900
  timeout $limit compute-sanitizer --tool $tool --error-exitcode 1 \
    python -m pytest tests/test_gpu_v2.py tests/test_gpu_kernels.py -m gpu -q -x -p no:cacheprovider \
    -k "(gram or topk or unbiased or ps_matches or qsvd or num_aggregate or full_rank or ps_update or qsgd or entrywise or bn) and not graph and not engine and not multi" \
    > gpurun_out/sanitizer_$tool.log 2>&1 || echo "$tool: exit $? (see gpurun_out/sanitizer_$tool.log)"
  tail -3 gpurun_out/sanitizer_$tool.log
done
