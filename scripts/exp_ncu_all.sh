#!/bin/bash
# ncu --set full of every hot kernel on one bin of 1.17e8 k-mers, with source counters; usage: exp_ncu_all.sh TAG [env assignments...]
set -u
OUT=${PROFILE_DIR:-profiles}          # where the report and the log go
mkdir -p "$OUT"
TAG=$1; shift
for kv in "$@"; do export "$kv"; done
timeout 900 ncu --set full --clock-control none --import-source on -k regex:"expand_kernel|walk_packs_parallel|msd_partition|msd_count|leaf_hash" -s 6 -c 6 -o $OUT/prof_all_${TAG} -f python scripts/probe_bin.py 117440512 31 2 > $OUT/ncu_all_${TAG}.log 2>&1
echo "ncu rc=$?"; tail -3 $OUT/ncu_all_${TAG}.log; ls -la $OUT/prof_all_${TAG}.ncu-rep
