#!/usr/bin/env bash
# A/B of the opt-in kernel variants (DESIGN.md §8, "prepared ... not yet run on a GPU") on one GPU:
#   1. the kernel-level tests of the variants (tests/test_zz_unverified_gpu.py),
#   2. bench.py once per switch setting; one JSON line per run in gpurun_out/ab_<name>.json.
# Usage (from the repo root, on the GPU box):  bash scripts/ab_switches.sh [steps] [warmup]
set -u
steps=${1:-6}
warmup=${2:-3}
out=gpurun_out
mkdir -p "$out"
# every opt-in test in its own process and under its own timeout: a hang or a sticky CUDA error in one of them must
# not hide the others (a timeout shows up as exit 124)
: > "$out/ab_tests.status"
hangs=0
for t in $(MER_RUN_UNVERIFIED=1 python -m pytest tests/test_zz_unverified_gpu.py --collect-only -q -p no:cacheprovider 2>/dev/null | grep "::"); do
  MER_RUN_UNVERIFIED=1 timeout -k 10 180 python -m pytest "$t" -q -x -p no:cacheprovider > "$out/ab_test_last.log" 2>&1
  rc=$?
  echo "$rc $t" | tee -a "$out/ab_tests.status"
  if [ $rc -ne 0 ]; then { echo "==== $t (exit $rc)"; tail -40 "$out/ab_test_last.log"; } >> "$out/ab_tests.log"; fi
  # three timeouts: stop spending GPU minutes on tests (and do not risk a wedged device); the bench lines still run
  if [ $rc -eq 124 ] || [ $rc -eq 137 ]; then hangs=$((hangs + 1)); fi
  if [ $hangs -ge 3 ]; then echo "3 timeouts: skipping the remaining opt-in tests" | tee -a "$out/ab_tests.status"; break; fi
done
run() {  # name, then VAR=value pairs
  local name=$1
  shift
  env "$@" python bench.py --steps "$steps" --warmup "$warmup" --cpu-clips 8 > "$out/ab_$name.json" 2> "$out/ab_$name.err"
  python - "$name" "$out/ab_$name.json" <<'PY'
import json, sys
name, path = sys.argv[1:3]
try:
    d = json.loads(open(path).read().strip().splitlines()[-1])
    other = {k["kernel"][:28]: round(k["frac"], 3) for k in d.get("roofline_other", [])}
    print(f"{name:16s} value {d['value']:8.1f} e2e {d['e2e']['value']:8.1f} ms/step {d['ms_per_step']:7.2f} "
          f"sm_mhz {d['clocks']['sm_mhz']} gemm_frac {d['roofline']['frac']:.3f} {other}")
except Exception as e:  # noqa: BLE001
    print(f"{name:16s} FAILED: {e}")
PY
}
run default MER_NOP=1
run att_short_off MER_ATT_SHORT=0
run att_short_all MER_ATT_SHORT=1
run gelu_packed MER_GELU_PACKED=1
run conv0_packed MER_CONV0_PACKED=1
run all_on MER_ATT_SHORT=1 MER_GELU_PACKED=1 MER_CONV0_PACKED=1
run default_again MER_NOP=1
# mixed-length audio: one pass per clip (default) against ragged batches
python scripts/bench_ragged_audio.py --clips 128 > "$out/ab_ragged_audio.jsonl" 2> "$out/ab_ragged_audio.err"
cat "$out/ab_ragged_audio.jsonl"
