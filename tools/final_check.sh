#!/bin/bash
# last check of the shipped defaults on one box: GPU tests, then the bench line (hard timeouts on both legs)
T=${1:-r02f}
O=tools_out
timeout -s KILL 330 python -m pytest tests -x -q -m gpu > $O/${T}_pytest_gpu.log 2>&1; tail -3 $O/${T}_pytest_gpu.log
timeout -s KILL 200 python bench.py --steps 30 --warmup 5 --skip-cpu-baseline > $O/${T}_bench_1gpu.json 2> $O/${T}_bench_1gpu.err; cut -c1-300 $O/${T}_bench_1gpu.json
