#!/bin/bash
# Round 2, call R: CTAs per SM of the latency kernel (PBSGPU_SPLIT_SPREAD_KB 30 -> 4, 85 -> 2) x size of its partition: fewer CTAs
# per SM run each chain faster.
mkdir -p gpurun_out
export CUDA_DEVICE_MAX_CONNECTIONS=32
PBSGPU_PARTITION_SMS=32 PBSGPU_SPLIT_SPREAD_KB=85 timeout 600 python -m pytest tests/test_gpu_round2.py tests/test_gpu_parity.py -q -x -k "cfg2 or early or async or knobs or partition or stream" > gpurun_out/r2r_pytest_p32s85.txt 2>&1; echo "pytest rc=$?" >> gpurun_out/r2r_pytest_p32s85.txt; tail -3 gpurun_out/r2r_pytest_p32s85.txt
run() {
  name=$1; shift
  env "$@" timeout 600 python bench.py --steps 20 --warmup 3 --no-e2e --no-cpu --no-verify > gpurun_out/r2r_$name.txt 2>gpurun_out/r2r_$name.err
  python - "$name" <<'PY' | tee -a gpurun_out/r2r_sweep.txt
import json, sys
n = sys.argv[1]
try:
    d = json.loads(open(f"gpurun_out/r2r_{n}.txt").read().strip().splitlines()[-1])
    v = d["value_distinct"]
    print(f"{n}: value {d['value']:.1f} GiB/s (K=20), value_distinct {v.get('value') or 0:.1f} GiB/s, single batch {d.get('single_batch_latency_ms', 0):.0f} ms", v.get("error", ""))
except Exception as ex:
    print(n, "failed", repr(ex))
PY
}
run A_p24_s30
run B_p32_s85 PBSGPU_PARTITION_SMS=32 PBSGPU_SPLIT_SPREAD_KB=85
run C_p40_s85 PBSGPU_PARTITION_SMS=40 PBSGPU_SPLIT_SPREAD_KB=85
run D_p24_s85 PBSGPU_PARTITION_SMS=24 PBSGPU_SPLIT_SPREAD_KB=85
run E_p32_s30 PBSGPU_PARTITION_SMS=32
