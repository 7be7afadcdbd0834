// tools/microbench.cu -- pipe-throughput and TMA-capability probes for design decisions
// (measurement aid, not product).  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench.bin tools/microbench.cu
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

enum { OP_SHF, OP_LOP3, OP_IADD3, OP_IMAD, OP_IMADHI, OP_PRMT, OP_MIX_LOP_IMAD, OP_MIX_SHF_IMADHI, OP_MIX_SHF_LOP, OP_MIX3, OP_COUNT };
static const char *OPNAME[] = {"SHF(rot)", "LOP3", "IADD3", "IMAD", "IMAD.HI", "PRMT", "LOP3+IMAD 1:1", "SHF+IMAD.HI 1:1", "SHF+LOP3 1:1", "SHF+LOP3+IMAD+IMAD 1:1:1:1"};

template <int OP>
__device__ __forceinline__ void op1(uint32_t &x, uint32_t a, uint32_t b, int k) {
    if (OP == OP_SHF) asm volatile("shf.r.wrap.b32 %0, %0, %0, %1;" : "+r"(x) : "r"(a));
    else if (OP == OP_LOP3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == OP_IADD3) asm volatile("{ .reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2; }" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == OP_IMAD) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == OP_IMADHI) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == OP_PRMT) asm volatile("prmt.b32 %0, %0, %1, %2;" : "+r"(x) : "r"(a), "r"(b));
    else if (OP == OP_MIX_LOP_IMAD) { if (k & 1) op1<OP_IMAD>(x, a, b, k); else op1<OP_LOP3>(x, a, b, k); }
    else if (OP == OP_MIX_SHF_IMADHI) { if (k & 1) op1<OP_IMADHI>(x, a, b, k); else op1<OP_SHF>(x, a, b, k); }
    else if (OP == OP_MIX_SHF_LOP) { if (k & 1) op1<OP_LOP3>(x, a, b, k); else op1<OP_SHF>(x, a, b, k); }
    else if (OP == OP_MIX3) { if ((k & 3) == 0) op1<OP_SHF>(x, a, b, k); else if ((k & 3) == 1) op1<OP_LOP3>(x, a, b, k); else op1<OP_IMAD>(x, a, b, k); }
}

template <int OP>
__global__ void k_pipe(uint32_t *out, uint32_t a, uint32_t b, int iters, long long *cyc) {
    uint32_t x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = threadIdx.x * 2654435761u + k;
    __syncthreads();
    long long t0 = clock64();
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int k = 0; k < 8; k++) op1<OP>(x[k], a, b, k);
    }
    long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= x[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int OP>
static void run_pipe(int sms, int warps_per_sm) {
    int threads = warps_per_sm * 32, iters = 4096;
    uint32_t *out; long long *cyc;
    CK(cudaMalloc(&out, (size_t)sms * threads * 4)); CK(cudaMalloc(&cyc, sms * 8));
    k_pipe<OP><<<sms, threads>>>(out, 7, 0x9e3779b9u, 64, cyc);
    CK(cudaDeviceSynchronize());
    k_pipe<OP><<<sms, threads>>>(out, 7, 0x9e3779b9u, iters, cyc);
    CK(cudaDeviceSynchronize());
    long long h[1024]; CK(cudaMemcpy(h, cyc, sms * 8, cudaMemcpyDeviceToHost));
    double avg = 0; for (int i = 0; i < sms; i++) avg += h[i]; avg /= sms;
    double ops = (double)threads * iters * 32;   // thread-ops per SM (IADD3 counts 1 per 2 adds)
    printf("  %-28s warps/SM %2d : %7.1f thread-ops/clk/SM\n", OPNAME[OP], warps_per_sm, ops / avg);
    cudaFree(out); cudaFree(cyc);
}

// ---------------------------------------------------------------------------------------------
// TMA tensor-map probe: byte-granular (unaligned) windows via overlapping rows
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

__global__ void k_tma2d(const __grid_constant__ CUtensorMap tmap, int c0, int c1, uint32_t bytes, uint8_t *out) {
    extern __shared__ __align__(128) uint8_t sm[];
    __shared__ __align__(8) uint64_t bar;
    uint32_t bar_s = (uint32_t)__cvta_generic_to_shared(&bar), dst = (uint32_t)__cvta_generic_to_shared(sm);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_s));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_s), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                     ::"r"(dst), "l"(&tmap), "r"(c0), "r"(c1), "r"(bar_s) : "memory");
    }
    asm volatile("{\n .reg .pred P1;\n W:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], 0;\n @P1 bra D;\n bra W;\n D:\n }" ::"r"(bar_s) : "memory");
    for (uint32_t i = threadIdx.x; i < bytes; i += blockDim.x) out[i] = sm[i];
}

static void tma_probe() {
    EncodeTiled enc = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void **)&enc, cudaEnableDefault, &qr) != cudaSuccess || !enc) {
        printf("TMA probe: cuTensorMapEncodeTiled not available\n"); return;
    }
    size_t N = 4 << 20;
    uint8_t *h = (uint8_t *)malloc(N), *d, *dout, *hout = (uint8_t *)malloc(16384);
    for (size_t i = 0; i < N; i++) h[i] = (uint8_t)((i * 2654435761u) >> 13);
    CK(cudaMalloc(&d, N)); CK(cudaMalloc(&dout, 16384)); CK(cudaMemcpy(d, h, N, cudaMemcpyHostToDevice));
    // (A) scan-style: rows of 512 B overlapping at stride 256, box 256 x 34 = 8704 contiguous bytes at any byte offset
    {
        CUtensorMap tm; cuuint64_t dims[2] = {512, N / 256 - 1}, strides[1] = {256}; cuuint32_t box[2] = {256, 34}, es[2] = {1, 1};
        CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        printf("TMA probe A (overlapping rows stride 256 / width 512, box 256x34): encode rc=%d\n", (int)r);
        if (r == CUDA_SUCCESS) {
            int offs[] = {0, 1, 3, 15, 16, 17, 100, 255, 256 * 7 + 5, 12345};
            int bad = 0;
            for (int oi = 0; oi < 10; oi++) {
                int p = offs[oi];
                CK(cudaFuncSetAttribute(k_tma2d, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384));
                k_tma2d<<<1, 128, 8704 + 128>>>(tm, p % 256, p / 256, 8704, dout);
                cudaError_t e = cudaDeviceSynchronize();
                if (e != cudaSuccess) { printf("   offset %d: launch failed %s\n", p, cudaGetErrorString(e)); bad++; break; }
                CK(cudaMemcpy(hout, dout, 8704, cudaMemcpyDeviceToHost));
                int ok = memcmp(hout, h + p, 8704) == 0;
                if (!ok) { bad++; printf("   offset %d: MISMATCH\n", p); }
            }
            printf("TMA probe A: %s\n", bad ? "FAILED" : "byte-granular 8704 B windows OK at all tested offsets");
        }
    }
    // (B) sha-style: long rows R+256 wide at stride R, box 256 x 1
    {
        cuuint64_t R = 1 << 20;
        CUtensorMap tm; cuuint64_t dims[2] = {R + 256, N / R - 1}, strides[1] = {R}; cuuint32_t box[2] = {256, 1}, es[2] = {1, 1};
        CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        printf("TMA probe B (rows R+256 wide at stride R=1MiB, box 256x1): encode rc=%d\n", (int)r);
        if (r == CUDA_SUCCESS) {
            size_t offs[] = {0, 5, 1000003, (1 << 20) - 100, (2 << 20) - 1, (2 << 20) + 77};
            int bad = 0;
            for (int oi = 0; oi < 6; oi++) {
                size_t p = offs[oi];
                k_tma2d<<<1, 128, 8704 + 128>>>(tm, (int)(p % R), (int)(p / R), 256, dout);
                cudaError_t e = cudaDeviceSynchronize();
                if (e != cudaSuccess) { printf("   offset %zu: launch failed %s\n", p, cudaGetErrorString(e)); bad++; break; }
                CK(cudaMemcpy(hout, dout, 256, cudaMemcpyDeviceToHost));
                if (memcmp(hout, h + p, 256) != 0) { bad++; printf("   offset %zu: MISMATCH\n", p); }
            }
            printf("TMA probe B: %s\n", bad ? "FAILED" : "byte-granular 256 B windows OK");
        }
    }
}

int main(int argc, char **argv) {
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    printf("device %s, %d SMs, cc %d.%d, smem/block optin %zu\n", p.name, p.multiProcessorCount, p.major, p.minor, p.sharedMemPerBlockOptin);
    int sms = p.multiProcessorCount;
    int wl[] = {4, 8, 16, 32};
    for (int wi = 0; wi < 4; wi++) {
        int w = wl[wi];
        run_pipe<OP_SHF>(sms, w); run_pipe<OP_LOP3>(sms, w); run_pipe<OP_IADD3>(sms, w); run_pipe<OP_IMAD>(sms, w);
        run_pipe<OP_IMADHI>(sms, w); run_pipe<OP_PRMT>(sms, w); run_pipe<OP_MIX_LOP_IMAD>(sms, w);
        run_pipe<OP_MIX_SHF_IMADHI>(sms, w); run_pipe<OP_MIX_SHF_LOP>(sms, w); run_pipe<OP_MIX3>(sms, w);
        printf("\n");
    }
    tma_probe();
    return 0;
}
