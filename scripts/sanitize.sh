#!/bin/bash
# compute-sanitizer passes over the kernel numerics checks (SURVEY.md 5.2: the reference has no race detection; we own
# streams, mbarrier / wgmma pipelines and peer-memory flags, so we need it).  Run on an H100:
#   scripts/sanitize.sh [memcheck|racecheck|synccheck|initcheck] [gpu_diag groups...]
# Small shapes only (the tools slow kernels 10-100x): DIAG_SMALL=1 makes gpu_diag skip its headline-shape timings.
set -u
cd "$(dirname "$0")/.."
TOOL=${1:-memcheck}; shift || true
GROUPS_=${*:-"elem gemm attn"}
LOGS=${DIAG_OUT:-diag_out}
mkdir -p "$LOGS"
for g in $GROUPS_; do
  echo "== compute-sanitizer --tool $TOOL : gpu_diag $g"
  DIAG_SMALL=1 timeout 900 compute-sanitizer --tool "$TOOL" --error-exitcode 66 --print-limit 20 \
      python scripts/gpu_diag.py "$g" > "$LOGS/sanitize_${TOOL}_${g}.log" 2>&1
  echo "   exit $? ; $(grep -c 'ERROR SUMMARY' "$LOGS/sanitize_${TOOL}_${g}.log") summary line(s): $(grep 'ERROR SUMMARY' "$LOGS/sanitize_${TOOL}_${g}.log" | tail -1)"
done
