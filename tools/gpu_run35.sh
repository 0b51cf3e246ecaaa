#!/bin/bash
# conv_tc2 consumer warpgroups taking MMA turns: parent vs turns on one card, arms alternated (ABBA).  Turns: named barriers 3 / 4
# (256 threads); per tap a consumer warpgroup bar.syncs on its own barrier before wgmma.fence, bar.arrives on the other's after
# wgmma.commit_group (before wait_group 0); warpgroup 1 arrives once before its work loop, warpgroup 0 syncs once before the exit.
# That schedule measured slower and is not in the tree: "change" here is a library built with it (_ab/lib_commit.so), _ab/libold.so the parent's
# (both git-ignored).  Usage: tools/gpu_run35.sh OUTDIR.  Results: profiles/r18_bench_ab.jsonl, profiles/r18_conv_layers_*.txt.
set -u
export OUT=$1
mkdir -p $OUT
O=$OUT/r18_log.txt
: > $O
CARD=$(nvidia-smi --query-gpu=name,power.limit --format=csv,noheader | head -n 1 | sed -E 's/, ([0-9]+)(\.[0-9]+)? W$/, \1 W power limit/')
echo "# card: $CARD" >> $O
cp _ab/lib_commit.so /tmp/lib_change.so
cp _ab/libold.so /tmp/lib_parent.so
use() { cp /tmp/lib_$1.so marconet_b200/libmarconet_b200.so; }
PYT="python -m pytest -q -p no:cacheprovider"

# 1. the kernel's own tests first: nothing else is worth running if they fail
use change
timeout 900 $PYT -m gpu tests/test_gpu_tc.py tests/test_gpu_tc_wide.py tests/test_gpu_conv_plan_space.py -x > $OUT/r18_tc_tests.txt 2>&1
rc=$?; tail -n 3 $OUT/r18_tc_tests.txt >> $O
if [ $rc -ne 0 ]; then echo "tensor-core tests failed ($rc)" >> $O; cat $O; exit 1; fi

# 2. bench A/B, 4 rounds per arm in ABBA order
CMD="bench.py --gpus 1 --steps 30 --warmup 5 --no-cpu-baseline --no-collective"
: > $OUT/r18_bench_ab.jsonl
round=0
for arm in parent change change parent parent change change parent; do
  use $arm
  timeout 600 python $CMD > $OUT/r18_bench_$arm.json 2> $OUT/r18_bench_$arm.err
  python - "$arm" "$CARD" "$CMD" >> $OUT/r18_bench_ab.jsonl <<'PY'
import os
import json, sys
arm, card, cmd = sys.argv[1:]
d = json.loads(open(os.environ["OUT"] + f"/r18_bench_{arm}.json").read().strip().splitlines()[-1])
print(json.dumps({"arm": "parent" if arm == "parent" else "this change", "value": d["value"], "ms_per_step": round(d["ms_per_step"], 3),
                  "card": card, "unit": d.get("unit", "chars/s"), "cmd": cmd}))
PY
done
python - >> $O <<'PY'
import os
import json, statistics
rows = [json.loads(l) for l in open(os.environ["OUT"] + "/r18_bench_ab.jsonl")]
seen = {}
for r in rows:
    seen[r["arm"]] = seen.get(r["arm"], 0) + 1
    r["round"] = seen[r["arm"]]
with open(os.environ["OUT"] + "/r18_bench_ab.jsonl", "w") as f:
    for r in rows:
        f.write(json.dumps({k: r[k] for k in ("arm", "round", "value", "ms_per_step", "card", "unit", "cmd")}) + "\n")
p = [r["value"] for r in rows if r["arm"] == "parent"]
c = [r["value"] for r in rows if r["arm"] == "this change"]
print("bench parent", p, "median", statistics.median(p))
print("bench change", c, "median", statistics.median(c))
print("median gain %.2f %%, min(change) > max(parent): %s" % (100 * (statistics.median(c) / statistics.median(p) - 1), min(c) > max(p)))
PY

# 3. the SR images of the timed step, both arms
for arm in parent change; do
  use $arm
  timeout 600 python bench.py --gpus 1 --steps 5 --warmup 2 --no-cpu-baseline --no-collective --dump-outputs /tmp/dump_$arm > /dev/null 2> $OUT/r18_dump_$arm.err
done
python - >> $O <<'PY'
import numpy as np
a, b = np.load("/tmp/dump_parent/sr.npy"), np.load("/tmp/dump_change/sr.npy")
print("sr.npy", a.shape, a.dtype, "array_equal:", bool(np.array_equal(a, b)), "max abs diff:", float(np.abs(a.astype(np.float64) - b).max()))
PY

# 4. per-layer tables, both arms, and their join
for arm in parent change; do
  use $arm
  MN_MODULE_GRAPHS=0 timeout 600 python tools/profile_conv_layers.py > $OUT/r18_conv_layers_$arm.txt 2>&1
  sed -i "1i # $CARD; MN_MODULE_GRAPHS=0 python tools/profile_conv_layers.py; library: $arm" $OUT/r18_conv_layers_$arm.txt
done
python - > $OUT/r18_conv_layers_ab.txt <<'PY'
import os
import re
pat = re.compile(r"^\s*([\d.]+) us\s+[\d.]+%\s+#(\d+)\s+(\S+)\s+(N\d+ \S+ \S+ k\d)\s+([\d.]+) TF\s+pipe\s+([\d.]+)\s+(.*)$")
def load(arm):
    out = {}
    for line in open(os.environ["OUT"] + f"/r18_conv_layers_{arm}.txt"):
        m = pat.match(line)
        if m:
            out[int(m.group(2))] = (float(m.group(1)), m.group(3), m.group(4), float(m.group(6)), m.group(7).strip())
    return out
p, c = load("parent"), load("change")
print("# per-layer A/B: event-timed eager calls, median of 10; gain = parent us / change us - 1")
print(f"{'#':>3s} {'layer':<40s} {'shape':<28s} {'plan':<12s} {'parent us':>9s} {'change us':>9s} {'pipe p':>6s} {'pipe c':>6s} {'gain':>7s}")
groups = {}
for s in sorted(p, key=lambda s: -p[s][0]):
    if s not in c:
        continue
    up, name, shape, pp, plan = p[s]
    uc, pc = c[s][0], c[s][3]
    print(f"{s:3d} {name:<40s} {shape:<28s} {plan:<12s} {up:9.1f} {uc:9.1f} {pp:6.2f} {pc:6.2f} {100 * (up / uc - 1):6.1f}%")
    g = plan.split()[0] if plan.startswith("tc") else "other"
    a = groups.setdefault(g, [0.0, 0.0, 0])
    a[0] += up; a[1] += uc; a[2] += 1
print()
for g, (up, uc, n) in sorted(groups.items()):
    print(f"{g:<10s} {n:3d} calls  parent {up:9.1f} us  change {uc:9.1f} us  gain {100 * (up / uc - 1):6.1f}%")
tp, tc = sum(v[0] for v in groups.values()), sum(v[1] for v in groups.values())
print(f"{'all':<10s} {sum(v[2] for v in groups.values()):3d} calls  parent {tp:9.1f} us  change {tc:9.1f} us  gain {100 * (tp / tc - 1):6.1f}%")
PY
tail -n 8 $OUT/r18_conv_layers_ab.txt >> $O

# 5. the whole GPU suite and smoke() on this change
use change
timeout 1500 $PYT -m gpu tests > $OUT/r18_pytest_gpu.txt 2>&1
echo "pytest -m gpu rc=$?" >> $O; tail -n 3 $OUT/r18_pytest_gpu.txt >> $O
timeout 300 python -c 'import __graft_entry__ as g; g.smoke()' > $OUT/r18_smoke.txt 2>&1
echo "smoke rc=$?" >> $O; tail -n 2 $OUT/r18_smoke.txt >> $O
use parent
cat $O
