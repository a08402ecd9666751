#!/usr/bin/env bash
# compute-sanitizer passes over the native kernels (needs an H100).
#   bash dev/sanitize.sh [memcheck|racecheck|synccheck|initcheck] [kernel-check name prefixes, comma separated]
# Each tool runs tests/gpu_kernel_check.py (every kernel against its fp32 reference) in --quick mode; racecheck and
# synccheck look at the shared-memory pipelines (mbarrier / TMA rings, epilogue staging slots), memcheck at global and
# peer-mapped accesses.  Expect a 10-50x slowdown: restrict with the second argument when iterating on one kernel.
set -euo pipefail
TOOL=${1:-memcheck}
ONLY=${2:-}
OUT=output/sanitize_${TOOL}.log
mkdir -p output
ARGS=(--quick --out output/sanitize_kernel_check.json)
if [ -n "$ONLY" ]; then ARGS+=(--only "$ONLY"); fi
timeout 1500 compute-sanitizer --tool "$TOOL" --error-exitcode 9 --print-limit 20 \
  python tests/gpu_kernel_check.py "${ARGS[@]}" > "$OUT" 2>&1 || echo "compute-sanitizer exit code $?"
grep -E "ERROR SUMMARY|RACECHECK SUMMARY|Error:|Hazard" "$OUT" | head -20
