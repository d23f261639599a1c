#!/bin/bash
# Environment-switch A/B of the whole step (graph-replayed), several repeats to see past the +-0.15 ms run-to-run noise.
# AB_CONFIGS lists the environments to compare, e.g. AB_CONFIGS="BASE=1 IH_PDL=0"; the default, BASE=1 alone, measures
# the run-to-run spread.
set -u
B="python bench.py --steps 20 --warmup 5 --no-cpu-baseline --no-eager-baseline --no-families"
for rep in 1 2; do
  for cfg in ${AB_CONFIGS:-"BASE=1"}; do
    v=$(env $cfg $B 2>/dev/null | tail -1 | python -c "import json,sys; d=json.loads(sys.stdin.read()); print(round(d['ms_per_step'],3), 'c1_512', round(d.get('c1_512',{}).get('ms_per_step',0),3))")
    echo "rep $rep $cfg ms_per_step $v"
  done
done
