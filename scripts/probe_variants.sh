#!/bin/bash
# GPU probe (not part of the test suite): the bench at 10 M reads under tuning switches; prints hash ms, pass 1 of both arms
# and the e2e step.  Usage: scripts/probe_variants.sh > probe.txt
for v in "ABB_TMA=1 ABB_H2D_OVERLAP=1" "ABB_TMA=0 ABB_H2D_OVERLAP=0"; do
  env $v python bench.py --reads 10000000 --steps 1 --warmup 1 --no-cpu-baseline 2>/dev/null | python -c "
import json,sys
d=json.loads(sys.stdin.read().strip().splitlines()[-1])
print('$v', 'step', round(d['ms_per_step'],1), 'hash', round(d['phases_ms']['hash'],1), 'pass1', round(d['pass1_ms'],1), 'e2e step', round(d['e2e']['ms_per_step'],1), 'e2e pass1', round(d['e2e']['pass1_ms'],1), d['fasta_md5'])
"
done
