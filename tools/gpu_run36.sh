#!/bin/bash
# Where the MMA hand-off between conv_tc2's consumer warpgroups goes (the turns of gpu_run35.sh), four libraries rotated:
# parent (no turns); commit: bar.arrive right after wgmma.commit_group; va: after wait_group 0, so one warpgroup's group is in the
# pipe at a time (ping-pong per tap); vc: the tap's 12 wgmmas in two commit groups (j = 0-1, 2-3), bar.arrive after wait_group 1.
# None is in the tree (git-ignored libraries _ab/lib_<arm>.so).  Usage: tools/gpu_run36.sh OUTDIR.  Results: profiles/r18_turn_variants.jsonl.
set -u
export OUT=$1
mkdir -p $OUT
O=$OUT/r18x_log.txt
: > $O
CARD=$(nvidia-smi --query-gpu=name,power.limit --format=csv,noheader | head -n 1 | sed -E 's/, ([0-9]+)(\.[0-9]+)? W$/, \1 W power limit/')
echo "# card: $CARD" >> $O
cp _ab/libold.so _ab/lib_parent.so
use() { cp _ab/lib_$1.so marconet_b200/libmarconet_b200.so; }
ARMS="va vc"
for arm in $ARMS; do
  use $arm
  timeout 600 python -m pytest -q -p no:cacheprovider -m gpu tests/test_gpu_tc.py tests/test_gpu_tc_wide.py tests/test_gpu_conv_plan_space.py -x > $OUT/r18x_tests_$arm.txt 2>&1
  echo "$arm tests rc=$? $(tail -n 1 $OUT/r18x_tests_$arm.txt)" >> $O
  timeout 300 python bench.py --gpus 1 --steps 5 --warmup 2 --no-cpu-baseline --no-collective --dump-outputs /tmp/dump_$arm > /dev/null 2>&1
done
use parent
timeout 300 python bench.py --gpus 1 --steps 5 --warmup 2 --no-cpu-baseline --no-collective --dump-outputs /tmp/dump_parent > /dev/null 2>&1
python - $ARMS >> $O <<'PY'
import sys, numpy as np
a = np.load("/tmp/dump_parent/sr.npy")
for arm in sys.argv[1:]:
    b = np.load(f"/tmp/dump_{arm}/sr.npy")
    print(arm, "sr.npy array_equal with parent:", bool(np.array_equal(a, b)))
PY
CMD="bench.py --gpus 1 --steps 30 --warmup 5 --no-cpu-baseline --no-collective"
: > $OUT/r18x_bench.jsonl
for rnd in 1 2 3; do
  for arm in parent commit va vc; do
    use $arm
    timeout 300 python $CMD > /tmp/b.json 2> /dev/null
    python -c "import json,sys; d=json.loads(open('/tmp/b.json').read().strip().splitlines()[-1]); print(json.dumps({'arm': sys.argv[1], 'round': int(sys.argv[2]), 'value': d['value'], 'ms_per_step': round(d['ms_per_step'], 3)}))" $arm $rnd >> $OUT/r18x_bench.jsonl
  done
done
python - >> $O <<'PY'
import os
import json, statistics
rows = [json.loads(l) for l in open(os.environ["OUT"] + "/r18x_bench.jsonl")]
p = statistics.median(r["value"] for r in rows if r["arm"] == "parent")
for arm in ("parent", "commit", "va", "vc"):
    v = [round(r["value"], 1) for r in rows if r["arm"] == arm]
    print(f"{arm:7s} {v} median {statistics.median(v):.1f} vs parent {100 * (statistics.median(v) / p - 1):+.2f} %")
PY
for arm in parent va vc; do
  use $arm
  MN_MODULE_GRAPHS=0 timeout 300 python tools/profile_conv_layers.py > $OUT/r18x_conv_layers_$arm.txt 2>&1
done
use parent
cat $O
