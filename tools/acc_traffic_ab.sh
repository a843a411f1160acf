#!/bin/sh
# Fused render kernel time with and without its accumulator-buffer traffic (SDB_AB_NO_ACC: the buffer is neither written
# nor read, results are wrong), on the same work: every sample of every live ray is marched, so the step count does not
# depend on the values.  Alternates the two builds; rebuilds the product library at the end.  Run from the repository root.
set -e
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader
for v in base no_acc base no_acc; do
    if [ "$v" = no_acc ]; then extra=-DSDB_AB_NO_ACC; else extra=; fi
    SDB_NVCC_EXTRA="$extra" python -m scenedreamer_b200.build --force > /dev/null
    python bench.py --gpus 1 --steps 5 --warmup 3 --no-cpu --no-extras --no-early-stop |
        python -c "import json, sys; d = json.loads(sys.stdin.read().strip().splitlines()[-1]); print('$v', 'kernel_ms %.1f' % d['roofline']['kernel_ms'], 'Msamples/s %.1f' % d['value'], 'clocks', d['clocks'])"
done
python -m scenedreamer_b200.build --force > /dev/null
