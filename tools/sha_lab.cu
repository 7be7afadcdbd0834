// tools/sha_lab.cu -- K3 instruction-mix laboratory (measurement aid, not product).
//
// SHA-256 on CUDA cores is bound by the two integer pipes of an SM sub-partition (ALU: SHF/LOP3/IADD3/PRMT/SEL,
// FMA: IMAD).
// This program times variants of the one-lane-per-range kernel that differ ONLY in which pipe their additions and
// logical shifts are sent to and in the launch shape, on N equal ranges (no length imbalance), and checks every
// digest against variant 0 (which is checked against a host SHA-256).  `tools/sass_mix.py` counts the loop's SASS
// per pipe for the same variants.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o tools/sha_lab.bin tools/sha_lab.cu
//   ./tools/sha_lab.bin mix [range_kib=256] [total_gib=16] [only_variant=-1]   instruction mixes at saturation
//   ./tools/sha_lab.bin load [chain_kib=1024]                                  chain latency and GB/s vs number of concurrent chains
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../pbs_plus_b200/csrc/sha256.cu"   // product kernels (k_sha_tuned, k_sha_split) for side-by-side timing, and their loader
using pbsgpu::ChunkRef;
using pbsgpu::ShaArgs;

#define CK(x) do { cudaError_t e__ = (x); if (e__ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e__), __LINE__); exit(1); } } while (0)

struct Opq { uint32_t one, p29, p22; };

__device__ __forceinline__ uint32_t rotr(uint32_t x, int r) { return __funnelshift_r(x, x, r); }
__device__ __forceinline__ uint32_t fadd(uint32_t a, uint32_t b, const Opq &o) {   // a + b on the FMA pipe: IMAD R, R, UR(=1), R
    uint32_t d; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(o.one), "r"(b)); return d;
}
__device__ __forceinline__ uint32_t fshr(uint32_t x, uint32_t pow2, const Opq &) {   // x >> n as mul.hi by 2^(32-n): IMAD.HI (half rate)
    uint32_t d; asm("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(pow2)); return d;
}

// variant bits: 1 = schedule additions on the FMA pipe, 2 = K+W on the FMA pipe, 4 = off-critical round additions
// (h+kw, d+h+kw) on the FMA pipe, 8 = ALL round additions on the FMA pipe (T = S1+ch shared), 16 = schedule shifts as IMAD.HI
template <int V>
__device__ __forceinline__ void compress(uint32_t (&st)[8], uint32_t (&w)[16], const Opq &o) {
    constexpr uint32_t K[64] = {K256_LIST};
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            const uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            const uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ ((V & 16) ? fshr(w15, o.p29, o) : (w15 >> 3));
            const uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ ((V & 16) ? fshr(w2, o.p22, o) : (w2 >> 10));
            if (V & 1) w[i & 15] = fadd(fadd(w[i & 15], s0, o), fadd(w[(i + 9) & 15], s1, o), o);
            else w[i & 15] = w[i & 15] + s0 + w[(i + 9) & 15] + s1;
        }
        const uint32_t kw = (V & 2) ? fadd(w[i & 15], K[i], o) : w[i & 15] + K[i];
        const uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
        const uint32_t ch = (e & f) ^ (~e & g);
        const uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
        const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t en, an;
        if (V & 8) {
            const uint32_t hk = fadd(h, kw, o), dhk = fadd(d, hk, o), t = fadd(S1, ch, o);
            en = fadd(dhk, t, o);
            an = fadd(fadd(fadd(S0, mj, o), hk, o), t, o);
        } else if (V & 4) {
            const uint32_t hk = fadd(h, kw, o), dhk = fadd(d, hk, o);
            en = S1 + ch + dhk;                 // IADD3
            const uint32_t x = S0 + mj + hk;    // IADD3
            an = x + S1 + ch;                   // IADD3
        } else {
            const uint32_t t1 = h + S1 + ch + kw, t2 = S0 + mj;
            en = d + t1; an = t1 + t2;
        }
        h = g; g = f; f = e; e = en; d = c; c = b; b = a; a = an;
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

__device__ __forceinline__ void sha_init(uint32_t (&s)[8]) {
    s[0] = 0x6a09e667; s[1] = 0xbb67ae85; s[2] = 0x3c6ef372; s[3] = 0xa54ff53a;
    s[4] = 0x510e527f; s[5] = 0x9b05688c; s[6] = 0x1f83d9ab; s[7] = 0x5be0cd19;
}

__device__ __noinline__ void finish(uint32_t (&s)[8], const uint8_t *tail, uint32_t rem, uint64_t len, uint8_t *out) {
    const uint64_t bits = len * 8;
    const int nblk = rem < 56 ? 1 : 2;
    Opq o{1u, 1u << 29, 1u << 22};
    for (int blk = 0; blk < nblk; blk++) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; i++) {
            uint32_t v = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint32_t idx = blk * 64 + i * 4 + k;
                uint32_t byte = idx < rem ? tail[idx] : (idx == rem ? 0x80u : 0u);
                v = (v << 8) | byte;
            }
            w[i] = v;
        }
        if (blk == nblk - 1) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
        compress<0>(s, w, o);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        out[4 * i] = (uint8_t)(s[i] >> 24); out[4 * i + 1] = (uint8_t)(s[i] >> 16);
        out[4 * i + 2] = (uint8_t)(s[i] >> 8); out[4 * i + 3] = (uint8_t)s[i];
    }
}

// one lane per range; the product's load path (pbsgpu::BlockStream, as in k_sha_tuned)
template <int V, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) k_lab(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                                       uint8_t *digests, Opq o) {
    const uint32_t t = blockIdx.x * THREADS + threadIdx.x;
    if (t >= n) return;
    const uint8_t *p = base + off[t];
    const uint64_t L = len[t];
    uint32_t s[8];
    sha_init(s);
    const uint32_t nblk = (uint32_t)(L >> 6);
    pbsgpu::BlockStream in(p, nblk);
    for (uint32_t b = 0; b < nblk; b++) {
        uint32_t w[16];
        in.next(b, w);
        compress<V>(s, w, o);
    }
    finish(s, p + (uint64_t)nblk * 64, (uint32_t)(L & 63), L, digests + (uint64_t)t * 32);
}

__global__ void k_fill(uint64_t *d, uint64_t nwords, uint64_t seed) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t z = seed + i * 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; d[i] = z ^ (z >> 31);
    }
}

// ---- host SHA-256 (check of variant 0) ----
static void host_sha256(const uint8_t *msg, size_t len, uint8_t out[32]) {
    static const uint32_t K[64] = {K256_LIST};
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    std::vector<uint8_t> m(msg, msg + len);
    m.push_back(0x80);
    while (m.size() % 64 != 56) m.push_back(0);
    for (int i = 7; i >= 0; i--) m.push_back((uint8_t)(((uint64_t)len * 8) >> (8 * i)));
    auto rr = [](uint32_t x, int r) { return (x >> r) | (x << (32 - r)); };
    for (size_t b = 0; b < m.size(); b += 64) {
        uint32_t w[64];
        for (int i = 0; i < 16; i++) w[i] = (m[b + 4 * i] << 24) | (m[b + 4 * i + 1] << 16) | (m[b + 4 * i + 2] << 8) | m[b + 4 * i + 3];
        for (int i = 16; i < 64; i++) w[i] = w[i - 16] + (rr(w[i - 15], 7) ^ rr(w[i - 15], 18) ^ (w[i - 15] >> 3)) + w[i - 7] + (rr(w[i - 2], 17) ^ rr(w[i - 2], 19) ^ (w[i - 2] >> 10));
        uint32_t a = h[0], bb = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
        for (int i = 0; i < 64; i++) {
            uint32_t t1 = hh + (rr(e, 6) ^ rr(e, 11) ^ rr(e, 25)) + ((e & f) ^ (~e & g)) + K[i] + w[i];
            uint32_t t2 = (rr(a, 2) ^ rr(a, 13) ^ rr(a, 22)) + ((a & bb) ^ (a & c) ^ (bb & c));
            hh = g; g = f; f = e; e = d + t1; d = c; c = bb; bb = a; a = t1 + t2;
        }
        h[0] += a; h[1] += bb; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }
    for (int i = 0; i < 8; i++) { out[4 * i] = h[i] >> 24; out[4 * i + 1] = h[i] >> 16; out[4 * i + 2] = h[i] >> 8; out[4 * i + 3] = h[i]; }
}

struct Work {
    const uint8_t *buf; const uint64_t *off, *len; uint32_t n; uint8_t *dig;
    const ChunkRef *refs; const unsigned long long *n_dev;   // product-kernel view of the same ranges
};
struct Variant { const char *name; void (*launch)(const Work &); };

template <int V, int THREADS, int MINB> static void lab(const Work &w) {
    Opq o{1u, 1u << 29, 1u << 22};
    k_lab<V, THREADS, MINB><<<(w.n + THREADS - 1) / THREADS, THREADS>>>(w.buf, w.off, w.len, w.n, w.dig, o);
}
static ShaArgs sha_args(const Work &w) {
    ShaArgs a; a.base = w.buf; a.off = nullptr; a.chunks = w.refs; a.order = nullptr; a.n_chunks = w.n_dev; a.chunk_cap = w.n;
    a.digests = w.dig; a.n_head = nullptr; a.part = 0; return a;
}
static void prod_tuned(const Work &w) {
    pbsgpu::Opq o{1u, 1u << 29, 1u << 22};
    pbsgpu::k_sha_tuned<false><<<(w.n + 31) / 32, 32>>>(sha_args(w), o, nullptr);
}
static void prod_split(const Work &w) {
    pbsgpu::Opq o{1u, 1u << 29, 1u << 22};
    pbsgpu::k_sha_split<false><<<(w.n + 31) / 32, 64>>>(sha_args(w), o, nullptr);
}

static const Variant VS[] = {
    {"v0   plain C (ptxas decides)         32 thr, <=72 regs", lab<0, 32, 28>},
    {"v3   sched adds + K+W on FMA         32 thr, <=72 regs", lab<3, 32, 28>},
    {"v7   v3 + off-critical round adds    32 thr, <=72 regs", lab<7, 32, 28>},
    {"v11  ALL adds on FMA                 32 thr, <=72 regs", lab<11, 32, 28>},
    {"v27  v11 + sched shifts IMAD.HI      32 thr, <=72 regs", lab<27, 32, 28>},
    {"v16  sched shifts IMAD.HI (= tuned)  32 thr, <=72 regs", lab<16, 32, 28>},
    {"v0                                   32 thr, <=64 regs", lab<0, 32, 32>},
    {"v11                                  32 thr, <=64 regs", lab<11, 32, 32>},
    {"v27                                  32 thr, <=64 regs", lab<27, 32, 32>},
    {"v0                                   32 thr, <=96 regs", lab<0, 32, 21>},
    {"v11                                  32 thr, <=96 regs", lab<11, 32, 21>},
    {"v0                                  128 thr, <=72 regs", lab<0, 128, 7>},
    {"v11                                 128 thr, <=72 regs", lab<11, 128, 7>},
    {"v27                                 128 thr, <=72 regs", lab<27, 128, 7>},
    {"v11                                 128 thr, <=64 regs", lab<11, 128, 8>},
    {"v27                                 128 thr, <=64 regs", lab<27, 128, 8>},
    {"v11                                 256 thr, <=64 regs", lab<11, 256, 4>},
    {"v27                                  64 thr, <=64 regs", lab<27, 64, 16>},
    {"v27                                 128 thr, <=56 regs", lab<27, 128, 9>},
    {"v11                                 128 thr, <=48 regs", lab<11, 128, 10>},
    {"v0                                  128 thr, <=48 regs", lab<0, 128, 10>},
    {"product k_sha_tuned", prod_tuned},
    {"product k_sha_split", prod_split},
};
static const int NV = (int)(sizeof VS / sizeof VS[0]);

struct Bench {
    uint8_t *buf = nullptr, *dig = nullptr, *dig0 = nullptr; uint64_t *d_off = nullptr, *d_len = nullptr; ChunkRef *d_refs = nullptr;
    unsigned long long *d_n = nullptr; uint64_t total = 0; uint32_t cap_n = 0;
    cudaEvent_t e0, e1;
    void init(uint64_t total_bytes, uint32_t max_n) {
        total = total_bytes; cap_n = max_n;
        CK(cudaMalloc(&buf, total + 4096)); CK(cudaMalloc(&dig, (size_t)max_n * 32)); CK(cudaMalloc(&dig0, (size_t)max_n * 32));
        CK(cudaMalloc(&d_off, (size_t)max_n * 8)); CK(cudaMalloc(&d_len, (size_t)max_n * 8)); CK(cudaMalloc(&d_refs, (size_t)max_n * sizeof(ChunkRef)));
        CK(cudaMalloc(&d_n, 8));
        k_fill<<<4096, 256>>>((uint64_t *)buf, (total + 4096) / 8, 77); CK(cudaDeviceSynchronize());
        CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    }
    // n equal ranges of `len` bytes at stride `stride`, misaligned by 3
    Work setup(uint32_t n, uint64_t stride, uint64_t len, std::vector<uint64_t> &off, std::vector<uint64_t> &ln) {
        off.resize(n); ln.resize(n); std::vector<ChunkRef> refs(n);
        for (uint32_t i = 0; i < n; i++) { off[i] = (uint64_t)i * stride + 3; ln[i] = len; refs[i].stream = 0; refs[i].len = (uint32_t)len; refs[i].start = off[i]; }
        unsigned long long hn = n;
        CK(cudaMemcpy(d_off, off.data(), (size_t)n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_len, ln.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(d_refs, refs.data(), (size_t)n * sizeof(ChunkRef), cudaMemcpyHostToDevice)); CK(cudaMemcpy(d_n, &hn, 8, cudaMemcpyHostToDevice));
        return Work{buf, d_off, d_len, n, dig, d_refs, d_n};
    }
    float time(const Variant &v, Work w, int reps) {
        CK(cudaMemset(w.dig, 0, (size_t)w.n * 32));
        v.launch(w); CK(cudaGetLastError()); CK(cudaDeviceSynchronize());
        float best = 1e9f;
        for (int r = 0; r < reps; r++) {
            CK(cudaEventRecord(e0)); v.launch(w); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
        }
        return best;
    }
};

int main(int argc, char **argv) {
    const char *mode = argc > 1 ? argv[1] : "mix";
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    printf("device %s, %d SMs, mode %s\n", prop.name, sms, mode);
    Bench B;
    std::vector<uint64_t> off, ln;
    if (!strcmp(mode, "mix")) {
        // saturation: every SM sub-partition has as many warps as the launch shape allows, equal ranges
        const uint64_t rk = argc > 2 ? atoll(argv[2]) : 256, tg = argc > 3 ? atoll(argv[3]) : 16;
        const int only = argc > 4 ? atoi(argv[4]) : -1;
        const uint64_t R = rk << 10; const uint32_t n = (uint32_t)((tg << 30) / R);
        B.init(tg << 30, n);
        Work w = B.setup(n, R, R - 64 + 5, off, ln);
        printf("%u ranges x %llu KiB\n", n, (unsigned long long)rk);
        std::vector<uint8_t> h0((size_t)n * 32), h1((size_t)n * 32);
        for (int v = 0; v < NV; v++) {
            if (only >= 0 && v != only && v != 0) continue;
            Work wv = w; if (v == 0) wv.dig = B.dig0;
            const float ms = B.time(VS[v], wv, 3);
            bool ok;
            if (v == 0) {
                CK(cudaMemcpy(h0.data(), B.dig0, (size_t)n * 32, cudaMemcpyDeviceToHost));
                std::vector<uint8_t> m(ln[5]); uint8_t ref[32];
                CK(cudaMemcpy(m.data(), B.buf + off[5], ln[5], cudaMemcpyDeviceToHost));
                host_sha256(m.data(), m.size(), ref);
                ok = memcmp(ref, &h0[5 * 32], 32) == 0;
            } else {
                CK(cudaMemcpy(h1.data(), B.dig, (size_t)n * 32, cudaMemcpyDeviceToHost));
                ok = memcmp(h0.data(), h1.data(), (size_t)n * 32) == 0;
            }
            printf("[%2d] %-56s %8.2f ms  %7.1f GB/s  %s\n", v, VS[v].name, ms, (double)n * ln[0] / ms / 1e6, ok ? "ok" : "MISMATCH");
            fflush(stdout);
        }
    } else if (!strcmp(mode, "load")) {
        // load curve: C concurrent chains of equal length; time per 64 B block of a chain = the chain latency that bounds
        // a batch's makespan, GB/s = throughput at that load.  C = 132 SMs x 4 sub-partitions x 32 lanes x {1/4 .. 8} warps.
        const uint64_t chain = (argc > 2 ? atoll(argv[2]) : 1024) << 10;   // bytes per chain
        int picks[5] = {0, 3, 4, -1, -1};                                       // v0, v11, v27, then the product kernels by name
        for (int v = 0; v < NV; v++) {
            if (!strcmp(VS[v].name, "product k_sha_tuned")) picks[3] = v;
            if (!strcmp(VS[v].name, "product k_sha_split")) picks[4] = v;
        }
        const uint32_t base_c = (uint32_t)sms * 4 * 32;
        const double mult[] = {0.25, 0.5, 1, 2, 4, 8};
        const uint32_t max_n = (uint32_t)(base_c * 8);
        B.init((uint64_t)max_n * chain > (64ull << 30) ? (64ull << 30) : (uint64_t)max_n * chain, max_n);
        printf("chains of %llu KiB; C chains = m x %u (one warp per sub-partition at m = 1)\n", (unsigned long long)(chain >> 10), base_c);
        for (int pi = (argc > 3 ? atoi(argv[3]) : 0); pi < 5; pi++) {
            for (int mi = 0; mi < 6; mi++) {
                const uint32_t n = (uint32_t)(base_c * mult[mi]);
                uint64_t len = chain; while ((uint64_t)n * len > B.total) len >>= 1;   // keep within the buffer
                Work w = B.setup(n, len, len - 64 + 5, off, ln);
                const float ms = B.time(VS[picks[pi]], w, 2);
                printf("%-40.40s C=%7u (m=%4.2f) len %5llu KiB: %8.2f ms  %7.1f GB/s  %6.3f us per 64 B block of a chain\n", VS[picks[pi]].name, n,
                       mult[mi], (unsigned long long)(len >> 10), ms, (double)n * ln[0] / ms / 1e6, ms * 1e3 / (double)(ln[0] / 64));
                fflush(stdout);
            }
        }
    }
    return 0;
}
