#!/bin/bash
# Round 2, call C: new tests, tuning sweep of the pipelined headline (slots / partition / threshold), distinct-data figure,
# stream bench, multi-rank test runs separately (--gpus 2).
mkdir -p gpurun_out
export CUDA_DEVICE_MAX_CONNECTIONS=32
timeout 900 python -m pytest tests -q -m gpu -x > gpurun_out/r2c_pytest_gpu.txt 2>&1; echo "pytest rc=$?" >> gpurun_out/r2c_pytest_gpu.txt; tail -5 gpurun_out/r2c_pytest_gpu.txt
B="python bench.py --steps 20 --warmup 3 --no-e2e --no-cpu --no-verify --no-distinct"
run() { name=$1; shift; env "$@" timeout 300 $B > gpurun_out/r2c_sweep_$name.txt 2>&1; python - "$name" <<'PY'
import json,re,sys
t=open(f"gpurun_out/r2c_sweep_{sys.argv[1]}.txt").read()
m=re.findall(r'\{.*\}',t)
if m:
    d=json.loads(m[-1]); print(sys.argv[1], round(d['value'],1), 'GiB/s', round(d['ms_per_step'],1), 'ms/step  iso', round(d['single_batch_latency_ms']), flush=True)
else: print(sys.argv[1], 'FAILED', t[-300:])
PY
}
run base X=1 | tee -a gpurun_out/r2c_sweep.txt
run slots8 PBSGPU_SLOTS=8 | tee -a gpurun_out/r2c_sweep.txt
run slots10 PBSGPU_SLOTS=10 | tee -a gpurun_out/r2c_sweep.txt
run slots15 PBSGPU_SLOTS=15 | tee -a gpurun_out/r2c_sweep.txt
run slots20 PBSGPU_SLOTS=20 | tee -a gpurun_out/r2c_sweep.txt
run slots26 PBSGPU_SLOTS=26 | tee -a gpurun_out/r2c_sweep.txt
run p32_t20_h64 PBSGPU_PARTITION_SMS=32 PBSGPU_HYBRID_THR_X10=20 PBSGPU_HYBRID_HEAD_PER_SM=64 | tee -a gpurun_out/r2c_sweep.txt
run p40_t15_h96 PBSGPU_PARTITION_SMS=40 PBSGPU_HYBRID_THR_X10=15 PBSGPU_HYBRID_HEAD_PER_SM=96 | tee -a gpurun_out/r2c_sweep.txt
run p32_t15_h128 PBSGPU_PARTITION_SMS=32 PBSGPU_HYBRID_THR_X10=15 PBSGPU_HYBRID_HEAD_PER_SM=128 | tee -a gpurun_out/r2c_sweep.txt
run p24_t20_h64 PBSGPU_HYBRID_THR_X10=20 PBSGPU_HYBRID_HEAD_PER_SM=64 | tee -a gpurun_out/r2c_sweep.txt
run p16 PBSGPU_PARTITION_SMS=16 | tee -a gpurun_out/r2c_sweep.txt
run lanes PBSGPU_SCAN_LANES=1 | tee -a gpurun_out/r2c_sweep.txt
run k32 X=1 | tee -a gpurun_out/r2c_sweep.txt
timeout 600 python bench.py --steps 20 --warmup 3 --no-e2e --no-cpu --no-verify > gpurun_out/r2c_bench_distinct.txt 2>&1; tail -c 1200 gpurun_out/r2c_bench_distinct.txt
timeout 600 python tools/stream_bench.py > gpurun_out/r2c_stream_bench.txt 2>&1; cat gpurun_out/r2c_stream_bench.txt
