#!/bin/bash
# Weight-ring depth of conv_tc2: parent (at most 4 weight stages) vs b6a (at most 6) vs b6b (at most 6, and a third A stage only
# when it leaves at least 4 weight stages), libraries _ab/lib_<arm>.so (git-ignored).  Usage: tools/gpu_run38.sh OUTDIR
set -u
OUT=$1
mkdir -p $OUT
O=$OUT/r19x_log.txt
: > $O
CARD=$(nvidia-smi --query-gpu=name,power.limit --format=csv,noheader | head -n 1 | sed -E 's/, ([0-9]+)(\.[0-9]+)? W$/, \1 W power limit/')
echo "# card: $CARD" >> $O
cp _ab/libold.so _ab/lib_parent.so
use() { cp _ab/lib_$1.so marconet_b200/libmarconet_b200.so; }
for arm in b6a b6b; do
  use $arm
  timeout 600 python -m pytest -q -p no:cacheprovider -m gpu tests/test_gpu_tc.py tests/test_gpu_tc_wide.py tests/test_gpu_conv_plan_space.py > $OUT/r19x_tests_$arm.txt 2>&1
  echo "$arm tests rc=$? $(tail -n 1 $OUT/r19x_tests_$arm.txt)" >> $O
done
CMD="bench.py --gpus 1 --steps 30 --warmup 5 --no-cpu-baseline --no-collective"
: > $OUT/r19x_bench.jsonl
for rnd in 1 2 3; do
  for arm in parent b6a b6b; do
    use $arm
    timeout 300 python $CMD > /tmp/b.json 2> /dev/null
    python -c "import json,sys; d=json.loads(open('/tmp/b.json').read().strip().splitlines()[-1]); print(json.dumps({'arm': sys.argv[1], 'round': int(sys.argv[2]), 'value': round(d['value'], 1), 'ms_per_step': round(d['ms_per_step'], 3)}))" $arm $rnd >> $OUT/r19x_bench.jsonl
  done
done
python - $OUT >> $O <<'PY'
import json, statistics, sys
rows = [json.loads(l) for l in open(sys.argv[1] + "/r19x_bench.jsonl")]
p = statistics.median(r["value"] for r in rows if r["arm"] == "parent")
for arm in ("parent", "b6a", "b6b"):
    v = [r["value"] for r in rows if r["arm"] == arm]
    print(f"{arm:7s} {v} median {statistics.median(v):.1f} vs parent {100 * (statistics.median(v) / p - 1):+.2f} %")
PY
for arm in parent b6a b6b; do
  use $arm
  MN_MODULE_GRAPHS=0 timeout 300 python tools/profile_conv_layers.py > $OUT/r19x_conv_layers_$arm.txt 2>&1
done
use parent
rm -f _ab/lib_parent.so
cat $O
