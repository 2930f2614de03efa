#!/bin/bash
# end-to-end variants of the bench (3 steps): the default, 4 slots.  prints value / e2e per setting
set -u
mkdir -p gpurun_out
for cfg in "" "KMCB200_E2E_SLOTS=4"; do
  ( for kv in $cfg; do export "$kv"; done; python bench.py --steps 3 --warmup 2 --no-cpu --no-secondary > gpurun_out/e2e_tmp.json 2> gpurun_out/e2e_tmp.err )
  python -c "
import json; d=json.load(open('gpurun_out/e2e_tmp.json')); print('%-28s value %.4g (%.1f ms)  e2e %.4g (%.1f ms)' % ('$cfg' or '(default)', d['value'], d['ms_per_step'], d['e2e']['value'], d['e2e']['ms_per_step']))" 2>&1 | tail -1
done
