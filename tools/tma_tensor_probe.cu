// tools/tma_tensor_probe.cu -- planning aid for K1's lane-contiguous variant.
//     nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/tma_tensor_probe.bin tools/tma_tensor_probe.cu
//     ./tools/tma_tensor_probe.bin
// Question: can ONE tensor-map TMA per warp step replace the 32 per-lane bulk copies of k_scan_lanes (which cost
// ~560 warp-instructions per step)?  The copy has to gather, for step k of a 64 KiB
// super-tile, the 256 B piece [L*2048 + k*256, +256) of every lane L and lay it out so that a quarter-warp's
// LDS.128 is bank-conflict free.
//   tensor map (u8): dim0 = 128 contiguous bytes, dim1 = 128 B unit index (stride 128: any 128 B aligned start),
//                    dim2 = lane 0..31 (stride 2048), dim3 = half 0..1 (stride 128); box {128, 1, 32, 2};
//                    SWIZZLE_128B.  Shared layout: [half][lane][128 B], 16 B chunk c of a row stored at c ^ (lane & 7).
// The probe (1) checks that cuTensorMapEncodeTiled accepts the overlapping strides, (2) verifies every byte a lane
// reads through the swizzled addressing against the byte pattern of the buffer, (3) times the copy-and-read loop
// against the one-contiguous-copy baseline of tma_piece_probe (mode 0 there: 4258 GB/s).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__host__ __device__ __forceinline__ uint8_t pattern(uint64_t a) { return (uint8_t)((a * 0x9E3779B97F4A7C15ull) >> 56); }

__device__ __forceinline__ uint32_t s32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n .reg .pred P1;\n W:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n @P1 bra D;\n bra W;\n D:\n }" ::"r"(bar), "r"(parity) : "memory");
}

__global__ void k_fill(uint8_t *d, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) d[i] = pattern(i);
}

constexpr int WARPS = 8, STEP_BYTES = 8192, SUPER = 65536;

template <bool VERIFY>
__global__ void __launch_bounds__(WARPS * 32, 1) k_probe(const __grid_constant__ CUtensorMap tmap, uint64_t bytes, uint32_t *sink,
                                                         unsigned long long *bad) {
    extern __shared__ __align__(1024) uint8_t sm[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *buf0 = sm + warp * 2 * STEP_BYTES;                       // 1024 B aligned (SWIZZLE_128B needs it)
    uint64_t *bars = (uint64_t *)(sm + WARPS * 2 * STEP_BYTES) + warp * 2;
    const uint32_t bar[2] = {s32(&bars[0]), s32(&bars[1])};
    if (lane == 0) {
        for (int i = 0; i < 2; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar[i]));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint64_t nsuper = bytes / SUPER, gw = (uint64_t)blockIdx.x * WARPS + warp, nw = (uint64_t)gridDim.x * WARPS;
    uint32_t acc = 0, uses[2] = {0, 0};
    unsigned long long wrong = 0;
    auto issue = [&](uint64_t st, int step, int b) {
        if (lane == 0) {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar[b]), "r"(STEP_BYTES) : "memory");
            const int c1 = (int)(st * (SUPER / 128) + step * 2);      // 128 B unit of lane 0's piece
            asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                         ::"r"(s32(buf0 + b * STEP_BYTES)), "l"(&tmap), "r"(0), "r"(c1), "r"(0), "r"(0), "r"(bar[b]) : "memory");
        }
    };
    for (uint64_t st = gw; st < nsuper; st += nw) {
        issue(st, 0, 0);
        for (int step = 0; step < 8; step++) {
            const int b = step & 1;
            if (step + 1 < 8) issue(st, step + 1, b ^ 1);
            bar_wait(bar[b], uses[b] & 1); uses[b]++;
            const uint8_t *buf = buf0 + b * STEP_BYTES;
#pragma unroll
            for (int c = 0; c < 16; c++) {                            // the lane's 256 B piece, 16 B at a time
                const int half = c >> 3, cc = c & 7;
                const uint4 v = *(const uint4 *)(buf + half * 4096 + lane * 128 + ((cc ^ (lane & 7)) << 4));
                acc ^= v.x ^ v.y ^ v.z ^ v.w;
                if (VERIFY) {
                    const uint64_t a0 = st * SUPER + (uint64_t)lane * 2048 + step * 256 + c * 16;
                    const uint8_t *pb = (const uint8_t *)&v;
                    for (int k = 0; k < 16; k++) wrong += pb[k] != pattern(a0 + k);
                }
            }
            __syncwarp();
        }
    }
    if (acc == 0x12345678u) sink[0] = acc;
    if (VERIFY && wrong) atomicAdd(bad, wrong);
}

typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
    const uint64_t bytes = 16ull << 30;
    uint8_t *d; uint32_t *sink; unsigned long long *bad;
    CK(cudaMalloc(&d, bytes)); CK(cudaMalloc(&sink, 4)); CK(cudaMalloc(&bad, 8)); CK(cudaMemset(bad, 0, 8));
    k_fill<<<4096, 256>>>(d, bytes); CK(cudaDeviceSynchronize());
    void *fn = nullptr; cudaDriverEntryPointQueryResult qr;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr));
    if (!fn || qr != cudaDriverEntryPointSuccess) { printf("cuTensorMapEncodeTiled not available\n"); return 1; }
    CUtensorMap tmap;
    const cuuint64_t dims[4] = {128, bytes / 128, 32, 2};
    const cuuint64_t strides[3] = {128, 2048, 128};                  // bytes, for dims 1..3 (overlapping on purpose)
    const cuuint32_t box[4] = {128, 1, 32, 2}, estr[4] = {1, 1, 1, 1};
    CUresult r = ((encode_fn)fn)(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, d, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    printf("cuTensorMapEncodeTiled(dims {128, n/128, 32, 2}, strides {128, 2048, 128}, box {128,1,32,2}, SWIZZLE_128B) -> %d\n", (int)r);
    if (r != CUDA_SUCCESS) { printf("encode rejected: try dim order {128, 32 (2048), 2 (128), n/128 (128)} next\n"); return 2; }
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    const int smem = WARPS * 2 * STEP_BYTES + WARPS * 2 * 8;
    CK(cudaFuncSetAttribute(k_probe<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(k_probe<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_probe<true><<<p.multiProcessorCount, WARPS * 32, smem>>>(tmap, 1ull << 30, sink, bad);
    CK(cudaDeviceSynchronize());
    unsigned long long hbad = 0; CK(cudaMemcpy(&hbad, bad, 8, cudaMemcpyDeviceToHost));
    printf("verify over 1 GiB: %llu wrong bytes (0 = the swizzled [half][lane][128 B] addressing is right)\n", hbad);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e9f;
    for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(e0);
        k_probe<false><<<p.multiProcessorCount, WARPS * 32, smem>>>(tmap, bytes, sink, bad);
        cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    printf("one 4-D tensor copy per warp step (32 x 256 B pieces, lane stride 2 KiB): %.2f ms, %.0f GB/s  (contiguous 8 KiB baseline: 4258 GB/s)\n",
           best, bytes / best / 1e6);
    return 0;
}
