#!/bin/bash
# A/B timing on ONE box: bench.py with several builds / option sets, alternating.
#   usage (on the GPU machine): bash tools/ab.sh <rounds> <steps> <variant>...     variant = <lib-suffix or "new">[:<PF_BENCH_OPTS>]
#   e.g. bash tools/ab.sh 2 10 base new new:pdl=0      (perspectivefields_b200/libpf_b200_<suffix>.so; "new" = the working-tree build)
R=${1:-2}; K=${2:-10}; shift 2
for i in $(seq $R); do
  for v in "$@"; do
    lib=${v%%:*}; opts=""; [[ "$v" == *:* ]] && opts=${v#*:}
    if [ "$lib" = new ]; then unset PF_B200_LIB; else export PF_B200_LIB=$PWD/perspectivefields_b200/libpf_b200_$lib.so; fi
    PF_BENCH_OPTS=$opts timeout 300 python bench.py --steps $K 2>/dev/null | tail -1 | python -c "import sys,json; d=json.loads(sys.stdin.read()); print('$v', round(d['value'],1), round(d['ms_per_step'],3), round(d['e2e']['value'],1), {k:round(x['ms_per_step'],2) for k,x in d['roofline']['per_engine'].items()})"
  done
done
