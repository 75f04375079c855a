# Multi-GPU validation of the owner-computes exchange: parity check, per-kernel profile, bench owner vs direct.
# usage (machine with N GPUs): [OUT=dir] bash tools/mgpu_validate.sh [N]   (results go to OUT, default a new temp dir)
N=${1:-2}
OUT=${OUT:-$(mktemp -d)}
mkdir -p "$OUT"
echo "results in $OUT"
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29511"
timeout 300 $TR tests/mgpu_xchg_check.py > "$OUT/xv_check.log" 2>&1; echo "check rc=$?"
tail -2 "$OUT/xv_check.log"
timeout 200 $TR tools/xchg_profile.py 2>&1 | grep '^{' | tee "$OUT/xv_prof.json"
for x in ${MODES:-owner direct}; do
  timeout 300 $TR bench.py --gpus $N --steps 50 --warmup 5 --exchange $x --no-cpu-baseline 2>&1 | grep '^{' > "$OUT/xv_${x}_$N.json"
  python - <<PY
import json
d = json.load(open("$OUT/xv_${x}_$N.json"))
print("$x", d["value"], d["ms_per_step"], d.get("e2e"))
PY
done
