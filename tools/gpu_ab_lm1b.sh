#!/bin/bash
# One-GPU A/B of the LM1B hot path: fused-op numerics, then the bench step under each
# environment "arm" (one switch flipped against the defaults per arm), then a per-stream kernel
# timeline of one replayed step.
# Run on one H100: bash tools/gpu_ab_lm1b.sh
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
timeout 200 python -m pytest tests/test_gpu_fused.py -x -q > gpurun_out/t_fused.log 2>&1; echo "fused_rc=$?"
tail -3 gpurun_out/t_fused.log
STEPS=${STEPS:-300}
ARMS=("default:" "head_unfused:PARALLAX_SSM_HEAD=0" "wpt_main:PARALLAX_LSTM_WPT_SIDE=0" \
      "nodbias:PARALLAX_LSTM_DBIAS_STREAM=0" "default2:")
for arm in "${ARMS[@]}"; do
  name=${arm%%:*}; envs=${arm#*:}
  env $envs timeout 90 python bench.py --no-extras --no-e2e --steps $STEPS --warmup 20 \
      > gpurun_out/ab_$name.json 2> gpurun_out/ab_$name.err
  python - "$name" <<'PY'
import json, sys
n = sys.argv[1]
try:
    d = json.loads(open("gpurun_out/ab_%s.json" % n).read().strip().splitlines()[-1])
    print("%-12s %.4f ms/step  %.0f words/s  launches %s" % (n, d["ms_per_step"], d["value"], d.get("gpu_launches")))
except Exception as e:
    print(n, "ERR", e)
PY
done
timeout 100 python tools/profile_step.py --graph --trace gpurun_out/trace_lm1b_r2b.txt \
    --out gpurun_out/profile_step_r2b.txt > gpurun_out/prof.log 2>&1; echo "prof_rc=$?"
