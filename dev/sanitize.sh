#!/usr/bin/env bash
# compute-sanitizer passes over the native kernels (needs an H100).
#   bash dev/sanitize.sh [memcheck|racecheck|synccheck|initcheck] [kernel-check name prefixes, comma separated]
#   bash dev/sanitize.sh [tool] tests/<gpu test file>[::test]
# Each tool runs tests/gpu_kernel_check.py (every kernel against its fp32 reference) in --quick mode; racecheck and
# synccheck look at the shared-memory pipelines (mbarrier / TMA rings, epilogue staging slots), memcheck at global and
# peer-mapped accesses.  Expect a 10-50x slowdown: restrict with the second argument when iterating on one kernel.
# A second argument naming a test file (e.g. tests/test_speculative_gpu.py::test_kernel_equals_the_mirror for the
# speculative acceptance kernel) runs that pytest selection under the tool instead.
set -euo pipefail
TOOL=${1:-memcheck}
ONLY=${2:-}
OUT=output/sanitize_${TOOL}.log
mkdir -p output
if [[ "$ONLY" == tests/*.py* ]]; then
  CMD=(python -m pytest -q -m gpu -p no:cacheprovider "$ONLY")
else
  CMD=(python tests/gpu_kernel_check.py --quick --out output/sanitize_kernel_check.json)
  if [ -n "$ONLY" ]; then CMD+=(--only "$ONLY"); fi
fi
timeout 1500 compute-sanitizer --tool "$TOOL" --error-exitcode 9 --print-limit 20 \
  "${CMD[@]}" > "$OUT" 2>&1 || echo "compute-sanitizer exit code $?"
grep -E "ERROR SUMMARY|RACECHECK SUMMARY|Error:|Hazard" "$OUT" | head -20
