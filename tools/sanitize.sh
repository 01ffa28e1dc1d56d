#!/bin/bash
# compute-sanitizer passes over the kernel diagnostics (SURVEY.md 5.2).  Run on a GPU box:
#   bash tools/sanitize.sh memcheck elementwise      bash tools/sanitize.sh racecheck bn      bash tools/sanitize.sh synccheck sgd
TOOL=${1:-memcheck}
GROUP=${2:-elementwise}
LOG=${SAN_LOG_DIR:-/tmp}/sanitize_${TOOL}_${GROUP}.log
timeout ${SAN_TIMEOUT:-900} compute-sanitizer --tool $TOOL --error-exitcode 3 --log-file $LOG \
    python tools/gpu_diag.py --group $GROUP
echo "compute-sanitizer $TOOL $GROUP rc=$?" | tee -a $LOG
tail -5 $LOG
