#!/bin/bash
# dev helper: A/B builds of libb200bpe.so (compile-time flags), each parity-tested and timed on the GPU box.
#   here (CPU):   bash tools/ab.sh build  name1:"-DFLAG=1" name2:"-DA=1 -DB=1" ...
#   on the GPU:   bash tools/ab.sh run [workloads...]     (every variant found in csrc/variants/)
set -u
CS=tiktoken_b200/csrc
if [ "$1" = build ]; then
  shift; mkdir -p $CS/variants; rm -f $CS/variants/*.so
  for spec in "$@"; do
    name=${spec%%:*}; flags=${spec#*:}; [ "$flags" = "$spec" ] && flags=""
    nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -shared -Xcompiler -fPIC $flags -o $CS/variants/libb200bpe_$name.so $CS/b200bpe.cu || exit 1
    echo "built $name ($flags)"
  done
  exit 0
fi
shift
OUT=$(mktemp -d); echo "logs in $OUT"
for so in $CS/variants/*.so; do
  name=$(basename $so .so); name=${name#libb200bpe_}
  export B200BPE_LIB=$PWD/$so
  timeout 600 python -m pytest tests/test_gpu_parity.py tests/test_gpu_paths.py -q -x -m gpu -k "not 200mib and not 256mib" > $OUT/ab_${name}_pytest.log 2>&1
  echo "== $name pytest rc=$? $(tail -1 $OUT/ab_${name}_pytest.log)"
  for spec in "${@:-config2}"; do
    w=${spec%%:*}; nb=${spec#*:}; [ "$nb" = "$spec" ] && nb=0
    timeout 300 python bench.py --workload $w --bytes $nb --steps 5 --warmup 3 --no-cpu-baseline --no-configs --no-extras 2>/dev/null | tail -1 > $OUT/ab_${name}_$w.json
    python - <<PY
import json
try:
    d=json.loads(open("$OUT/ab_${name}_$w.json").read()); s=d["stage_ms"]
    print("   $w", round(d["value"],1),"GB/s", round(d["ms_per_step"],3),"ms e2e", round(d["e2e"]["value"],1), {k[:-3]: round(v,3) for k,v in s.items()})
except Exception as e: print("   $w failed", e)
PY
  done
done
