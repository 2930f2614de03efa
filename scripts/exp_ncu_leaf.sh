#!/bin/bash
# one ncu --set full capture of the leaf kernel (bin of 1.17e8 k-mers), with source counters; usage: exp_ncu_leaf.sh TAG [env assignments...]
set -u
OUT=${PROFILE_DIR:-profiles}          # where the report and the log go
mkdir -p "$OUT"
TAG=$1; shift
for kv in "$@"; do export "$kv"; done
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"leaf_hash" -s 2 -c 1 -o $OUT/prof_leaf_${TAG} -f python scripts/probe_bin.py 117440512 31 2 > $OUT/ncu_leaf_${TAG}.log 2>&1
echo "ncu rc=$?"; tail -3 $OUT/ncu_leaf_${TAG}.log; ls -la $OUT/prof_leaf_${TAG}.ncu-rep
