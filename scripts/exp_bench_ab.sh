#!/bin/bash
# A/B runs of bench.py (diagnosis only): each line = variant, value, ms/step of the device-resident
# region, ms/step of the end-to-end region, sum of the timed spans per step.
mkdir -p gpurun_out
run() {
  name=$1; shift
  env "$@" timeout 400 python bench.py --steps 6 --warmup 3 > gpurun_out/exp_$name.json 2> gpurun_out/exp_$name.err
  python - <<PY
import json
d = json.load(open("gpurun_out/exp_$name.json"))
k = d["kernels"]
print("$name", d["value"], d["ms_per_step"], "e2e", d["e2e"]["ms_per_step"], "spans/step",
      round(sum(v["ms"] for v in k.values()) / d["steps"], 1), "host", d.get("host_enqueue_ms_per_step"),
      d.get("allocator_in_timed_region"), d["clocks"].get("sm_mhz"))
PY
}
for v in "$@"; do
  case $v in
    A) run A X=1 ;;
    NOSAMPLER) run NOSAMPLER LLMC_BENCH_SAMPLER=0 ;;
    NOTIMER) run NOTIMER LLMC_BENCH_TIMER=0 ;;
    SYNC) run SYNC LLMC_BENCH_STEP_SYNC=1 ;;
    NOTIMER_SYNC) run NOTIMER_SYNC LLMC_BENCH_TIMER=0 LLMC_BENCH_STEP_SYNC=1 ;;
    EXPAND) run EXPAND PYTORCH_CUDA_ALLOC_CONF=expandable_segments:True ;;
  esac
done
