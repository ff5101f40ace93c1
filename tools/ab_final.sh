#!/bin/bash
# A/B of the cluster split-K variants on one box; every leg under its own hard timeout
# (a hung leg must not take the rest of the call with it).  Outputs under tools_out/.
T=${1:-r02e}
O=tools_out
timeout -s KILL 330 python -m pytest tests -x -q -m gpu > $O/${T}_pytest_gpu.log 2>&1; tail -3 $O/${T}_pytest_gpu.log
run() {   # name, env assignments...
    local name=$1; shift
    timeout -s KILL 170 env "$@" python bench.py --steps 30 --warmup 5 --skip-cpu-baseline > $O/${T}_bench_${name}.json 2> $O/${T}_bench_${name}.err
    echo "$name rc=$? $(cut -c1-230 $O/${T}_bench_${name}.json)"
}
run default CB_NOOP=1
run cluster_sk_lane0 CB_GEMM_CLUSTER_SK=1
run cluster_sk_all CB_GEMM_CLUSTER_SK=2
