#!/bin/bash
# Sanity run on one H100: the whole GPU test tier, smoke(), the default bench line and
# a kernel timeline of one replayed LM1B step.
# bash tools/gpu_final_check.sh
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
timeout 240 python -m pytest tests -m gpu -x -q > gpurun_out/pytest_gpu_final.log 2>&1; echo "pytest_rc=$?"
tail -2 gpurun_out/pytest_gpu_final.log
timeout 90 python __graft_entry__.py --smoke > gpurun_out/smoke_final.log 2>&1; echo "smoke_rc=$?"
tail -1 gpurun_out/smoke_final.log
timeout 60 python tools/profile_step.py --graph --trace gpurun_out/trace_lm1b_r2c.txt \
    --out gpurun_out/profile_step_r2c.txt > gpurun_out/prof.log 2>&1; echo "prof_rc=$?"
timeout 240 python bench.py > gpurun_out/bench_lm1b_1gpu_final.json 2> gpurun_out/bench_final.err; echo "bench_rc=$?"
python - <<'PY'
import json
d = json.loads(open("gpurun_out/bench_lm1b_1gpu_final.json").read().strip().splitlines()[-1])
print(d["ms_per_step"], d["value"], d.get("e2e"), d.get("gpu_launches"), d.get("clocks"))
PY
