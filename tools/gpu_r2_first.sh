#!/bin/bash
# First gpurun call of round 2 (everything round 1 could not fit into its GPU budget), ~6-8 GPU-minutes:
#   1. the whole GPU suite + smoke on HEAD,
#   2. the tensor-map TMA probe that decides how K1's lane-contiguous variant is rebuilt (DESIGN.md 5c item 2),
#   3. ncu --set full of K7 phase A (k_xxh3_blocks) and phase B (k_xxh3_chain): dram bytes, pipe utilisation,
#   4. a short bench line (headline + the K7 figure in next_rows).
# Read afterwards: gpurun_out/r2_*.txt ; python tools/ncu_summary.py gpurun_out/prof_xxh3.ncu-rep
mkdir -p gpurun_out
export CUDA_DEVICE_MAX_CONNECTIONS=32
timeout 900 python -m pytest tests -x -q -m gpu > gpurun_out/r2_pytest_gpu.txt 2>&1; echo "pytest rc=$?" >> gpurun_out/r2_pytest_gpu.txt; tail -3 gpurun_out/r2_pytest_gpu.txt
timeout 300 python __graft_entry__.py smoke 2>&1 | tail -1 | tee gpurun_out/r2_smoke.txt
[ -x tools/tma_tensor_probe.bin ] || nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/tma_tensor_probe.bin tools/tma_tensor_probe.cu
timeout 120 ./tools/tma_tensor_probe.bin 2>&1 | tee gpurun_out/r2_tma_tensor_probe.txt
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_xxh3_ -c 2 -f -o gpurun_out/prof_xxh3 \
    python tools/xxh3_bench.py 8 > gpurun_out/r2_ncu_xxh3.log 2>&1; tail -2 gpurun_out/r2_ncu_xxh3.log
timeout 600 python bench.py --steps 16 --warmup 3 --no-cpu > gpurun_out/r2_bench.txt 2>&1; tail -c 600 gpurun_out/r2_bench.txt
