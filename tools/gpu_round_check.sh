#!/bin/bash
# One GPU-box pass over the round's evidence: smoke, device timings, bench line, GPU tests.
# usage: tools/gpu_round_check.sh <tag> [configs for tools/time_configs.py ...]
TAG=${1:-r2}; shift
OUT=gpurun_out/$TAG; mkdir -p $OUT
python -c "import __graft_entry__ as g; g.build(); g.smoke()" > $OUT/smoke.log 2>&1; echo "smoke rc=$?"
timeout 600 python tools/time_configs.py "$@" > $OUT/time_configs.txt 2>&1; echo "time_configs rc=$?"; cat $OUT/time_configs.txt
timeout 900 python bench.py > $OUT/bench.json 2> $OUT/bench.err; echo "bench rc=$?"; cut -c1-1500 $OUT/bench.json
timeout 1200 python -m pytest tests -m gpu -x -q > $OUT/pytest_gpu.log 2>&1; echo "pytest rc=$?"; tail -5 $OUT/pytest_gpu.log
