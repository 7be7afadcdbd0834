#!/bin/bash
# Round 2, call A: whole GPU suite on HEAD (incl. the round-2 tests), SHA instruction-mix lab, tensor-map probe,
# ncu --set full of K7 / K6 / saturated K3 (modes 0,1,3), one full bench line.
mkdir -p gpurun_out
export CUDA_DEVICE_MAX_CONNECTIONS=32
nvidia-smi --query-gpu=name,clocks.max.sm,power.limit --format=csv | tee gpurun_out/r2a_gpu.txt; nproc >> gpurun_out/r2a_gpu.txt
timeout 1500 python -m pytest tests -q -m gpu > gpurun_out/r2a_pytest_gpu.txt 2>&1; echo "pytest rc=$?" >> gpurun_out/r2a_pytest_gpu.txt; tail -15 gpurun_out/r2a_pytest_gpu.txt
[ -x tools/sha_lab.bin ] || nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o tools/sha_lab.bin tools/sha_lab.cu
timeout 300 ./tools/sha_lab.bin mix 256 16 > gpurun_out/r2a_sha_lab_mix.txt 2>&1; cat gpurun_out/r2a_sha_lab_mix.txt
timeout 400 ./tools/sha_lab.bin load 1024 > gpurun_out/r2a_sha_lab_load.txt 2>&1; tail -40 gpurun_out/r2a_sha_lab_load.txt
for l in 0 1; do for part in 24 0; do
  PBSGPU_SCAN_LANES=$l PBSGPU_PARTITION_SMS=$part timeout 200 python tools/scan_bench.py 32 2>&1 | tail -1 | tee -a gpurun_out/r2a_scan_bench.txt
done; done
[ -x tools/tma_tensor_probe.bin ] || nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/tma_tensor_probe.bin tools/tma_tensor_probe.cu
timeout 120 ./tools/tma_tensor_probe.bin 2>&1 | tee gpurun_out/r2a_tma_tensor_probe.txt
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_xxh3_ -c 2 -f -o gpurun_out/prof_xxh3 \
    python tools/xxh3_bench.py 8 > gpurun_out/r2a_ncu_xxh3.log 2>&1; tail -2 gpurun_out/r2a_ncu_xxh3.log
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_crc32 -c 1 -f -o gpurun_out/prof_crc32 \
    python tools/crc_bench.py > gpurun_out/r2a_ncu_crc.log 2>&1; tail -2 gpurun_out/r2a_ncu_crc.log
# saturated K3 through the lab binary (variant indices: 0 = v0, 3 = v11, 4 = v27), 32 Ki ranges x 1 MiB = full occupancy for the whole capture
for v in 0 3 4; do
  skip=6; [ $v -eq 0 ] && skip=2      # with a variant selected the lab runs v0 first (4 launches) as the digest reference
  timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_lab --launch-skip $skip -c 1 -f \
      -o gpurun_out/prof_lab_sat_$v ./tools/sha_lab.bin mix 1024 32 $v > gpurun_out/r2a_ncu_lab_$v.log 2>&1; tail -1 gpurun_out/r2a_ncu_lab_$v.log
done
timeout 900 python bench.py --steps 20 --warmup 3 > gpurun_out/r2a_bench.txt 2>gpurun_out/r2a_bench.err; tail -c 2500 gpurun_out/r2a_bench.txt; tail -5 gpurun_out/r2a_bench.err
