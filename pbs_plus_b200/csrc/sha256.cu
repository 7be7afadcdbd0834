// pbs_plus_b200/csrc/sha256.cu -- K3: batched per-chunk SHA-256 (FIPS 180-4), sm_90a.
//
// Replaces the per-chunk digest the reference's dedup writer computes for every chunk
// cut inside transfer.ArchiveWriter.WriteEntryReader (reference
// internal/pxarmount/commit.go:720, :858; CryptModeNone commit.go:314 => plain SHA-256
// of the raw chunk bytes; Go crypto/sha256 in the reference build).
//
// SHA-256 is a serial chain per message, so the parallelism is ACROSS chunks: one lane
// per chunk, chunks taken longest-first (K2's chunks sorted by length) so that the 32
// lanes of a warp retire together and the longest chunks start first.  Integer work on
// the ALU/FMA pipes; no tensor cores.  The kernel is instruction bound (~22 integer
// ops per byte), not HBM bound -- see DESIGN.md for the ceiling this implies.
#include <cuda_runtime.h>
#include <stdint.h>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

// compile-time copy so that fully unrolled rounds take K as an immediate operand
#define K256_LIST                                                                                          \
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,        \
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,        \
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,        \
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,        \
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,        \
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,        \
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,        \
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2

__device__ __forceinline__ uint32_t rotr(uint32_t x, int r) { return __funnelshift_r(x, x, r); }

struct Sha256State { uint32_t h[8]; };

__device__ __forceinline__ void sha_init(Sha256State &s) {
    s.h[0] = 0x6a09e667; s.h[1] = 0xbb67ae85; s.h[2] = 0x3c6ef372; s.h[3] = 0xa54ff53a;
    s.h[4] = 0x510e527f; s.h[5] = 0x9b05688c; s.h[6] = 0x1f83d9ab; s.h[7] = 0x5be0cd19;
}

// One compression: w[16] = big-endian message words (clobbered).
__device__ __forceinline__ void sha_compress(Sha256State &s, uint32_t (&w)[16]) {
    constexpr uint32_t K[64] = {K256_LIST};
    uint32_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
            uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
            w[i & 15] = w[i & 15] + s0 + w[(i + 9) & 15] + s1;
        }
        uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
        uint32_t ch = (e & f) ^ (~e & g);
        uint32_t t1 = h + S1 + ch + K[i] + w[i & 15];
        uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
        uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t t2 = S0 + mj;
        h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}

// Padding blocks for a message of `len` bytes whose unprocessed tail (rem = len % 64
// bytes) starts at `tail`.
__device__ __noinline__ void sha_finish(Sha256State &s, const uint8_t *tail, uint32_t rem, uint64_t len, uint8_t *out) {
    const uint64_t bits = len * 8;
    const int nblk = rem < 56 ? 1 : 2;
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
        sha_compress(s, w);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        out[4 * i] = (uint8_t)(s.h[i] >> 24); out[4 * i + 1] = (uint8_t)(s.h[i] >> 16);
        out[4 * i + 2] = (uint8_t)(s.h[i] >> 8); out[4 * i + 3] = (uint8_t)s.h[i];
    }
}

// sha_finish of the keyed message (chunk || suffix[32]) of encrypt mode: the 32 suffix bytes follow the tail, so only
// these final one or two blocks differ from the plain digest's.  A function of its own, so sha_finish and the kernels that
// call it keep their code.
__device__ __noinline__ void sha_finish_keyed(Sha256State &s, const uint8_t *tail, uint32_t rem, uint64_t len,
                                              const uint8_t *suffix, uint8_t *out) {
    const uint64_t bits = (len + 32) * 8;
    const uint32_t end = rem + 32;
    const int nblk = end < 56 ? 1 : 2;
    for (int blk = 0; blk < nblk; blk++) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; i++) {
            uint32_t v = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint32_t idx = blk * 64 + i * 4 + k;
                uint32_t byte = idx < rem ? tail[idx] : idx < end ? suffix[idx - rem] : (idx == end ? 0x80u : 0u);
                v = (v << 8) | byte;
            }
            w[i] = v;
        }
        if (blk == nblk - 1) { w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits; }
        sha_compress(s, w);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        out[4 * i] = (uint8_t)(s.h[i] >> 24); out[4 * i + 1] = (uint8_t)(s.h[i] >> 16);
        out[4 * i + 2] = (uint8_t)(s.h[i] >> 8); out[4 * i + 3] = (uint8_t)s.h[i];
    }
}
// the digest of a hash whose full blocks are done: plain, or keyed with `suffix`
template <bool KEYED>
__device__ __forceinline__ void sha_done(const ShaArgs &a, const uint8_t *suffix, Sha256State &s, const uint8_t *tail,
                                         const ChunkRef &c, uint32_t id) {
    if (KEYED) sha_finish_keyed(s, tail, c.len & 63, c.len, suffix, a.digests + (uint64_t)id * 32);
    else sha_finish(s, tail, c.len & 63, c.len, a.digests + (uint64_t)id * 32);
}

// 64 message bytes at arbitrary alignment -> 16 big-endian words.
// Loads 4-byte aligned words; ONE PRMT per word does the realignment and the byte swap.
__device__ __forceinline__ void load_block_be(const uint8_t *p, uint32_t (&w)[16]) {
    const uint32_t sh = (uint32_t)((uintptr_t)p & 3);
    const uint32_t *q = (const uint32_t *)(p - sh);
    // bytes of {lo,hi} are indexed 0..7; big-endian word = bytes sh, sh+1, sh+2, sh+3
    const uint32_t sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
    uint32_t x[17];
#pragma unroll
    for (int i = 0; i < 16; i++) x[i] = __ldg(q + i);
    x[16] = sh ? __ldg(q + 16) : 0;   // never touch the word past the block when aligned
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = __byte_perm(x[i], x[i + 1], sel);
}

// ---------------------------------------------------------------------------
// The full blocks of one hash as 16-byte aligned LDG.128 loads (5 per 64 B block instead of 17 LDG.32: the L1/tex path
// is charged per distinct line per instruction, so wide loads matter even though the kernels are ALU bound), the next
// block prefetched while the current one is compressed; the per-lane word misalignment is undone by a 2-stage SEL
// network and the byte misalignment + endian swap by ONE PRMT per word.  A hash of `len` bytes at p reads the vec_count
// aligned vectors from first_vec(p) and no others (the blocks here, the tail in sha_finish); the arena copies just these.
// ---------------------------------------------------------------------------
struct BlockStream {
    static __device__ __forceinline__ const uint4 *first_vec(const uint8_t *p) { return (const uint4 *)(p - ((uintptr_t)p & 15)); }
    // bytes from first_vec(p) to the end of the input; vec_count rounds it up to whole vectors
    static __device__ __forceinline__ uint64_t vec_span(const uint8_t *p, uint32_t len) { return ((uintptr_t)p & 15) + (uint64_t)len; }
    static __device__ __forceinline__ uint64_t vec_count(const uint8_t *p, uint32_t len) { return (vec_span(p, len) + 15) >> 4; }

    uint4 v4, v3, v2, v1, v0;   // declared first and in this order, they keep k_sha_tuned's SASS that of an inline loader
    const uint4 *q;
    uint32_t nblk, sel;
    bool need5, d1, d2;

    // `nblk` full blocks at p; issues the loads of block 0
    __device__ __forceinline__ BlockStream(const uint8_t *p, uint32_t nblk_) : nblk(nblk_) {
        const uint32_t delta = (uint32_t)((uintptr_t)p & 15), dw = delta >> 2, sh = delta & 3;
        q = (const uint4 *)(p - delta);
        sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
        need5 = delta != 0;     // never touch the vector past the block when the chunk is 16 B aligned
        d1 = dw & 1; d2 = dw & 2;
        v4 = make_uint4(0, 0, 0, 0);
        if (nblk) {
            v0 = __ldg(q); v1 = __ldg(q + 1); v2 = __ldg(q + 2); v3 = __ldg(q + 3);
            if (need5) v4 = __ldg(q + 4);
        }
    }
    // block b's 16 big-endian words; issues the loads of block b + 1
    __device__ __forceinline__ void next(uint32_t b, uint32_t (&w)[16]) {
        uint32_t x[20] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w,
                          v3.x, v3.y, v3.z, v3.w, v4.x, v4.y, v4.z, v4.w};
        if (b + 1 < nblk) {                     // v4 of this block == v0 of the next
            const uint4 *qn = q + (uint64_t)(b + 1) * 4;
            v0 = need5 ? v4 : __ldg(qn);
            v1 = __ldg(qn + 1); v2 = __ldg(qn + 2); v3 = __ldg(qn + 3);
            if (need5) v4 = __ldg(qn + 4);
        }
        uint32_t y[18];
#pragma unroll
        for (int i = 0; i < 18; i++) y[i] = d2 ? x[i + 2] : x[i];
#pragma unroll
        for (int i = 0; i < 17; i++) y[i] = d1 ? y[i + 1] : y[i];
#pragma unroll
        for (int i = 0; i < 16; i++) w[i] = __byte_perm(y[i], y[i + 1], sel);
    }
};

// The chunk at position t of `order`: its id (which indexes its digest) and ChunkRef; returns its first byte in the source.
__device__ __forceinline__ const uint8_t *sha_chunk(const ShaArgs &a, uint64_t t, uint32_t &id, ChunkRef &c) {
    id = a.order ? a.order[t] : (uint32_t)t;
    c = a.chunks[id];
    return a.base + (a.off ? a.off[c.stream] : 0) + c.start;
}

// position in `order` handled by logical thread t of a launch, honouring the hybrid split
__device__ __forceinline__ bool sha_slot(const ShaArgs &a, uint64_t t, uint64_t &pos) {
    const unsigned long long n = live_count(*a.n_chunks, a.chunk_cap);
    const unsigned long long head = live_count(a.part ? *a.n_head : 0ull, n);
    if (a.part == 1) { pos = t; return t < head; }
    pos = t + head;
    return pos < n;
}

// ---------------------------------------------------------------------------
// Cross-check / v0 kernel: one thread per chunk, chunks in `order` (longest first).
// ---------------------------------------------------------------------------
template <bool KEYED>
__device__ __forceinline__ void sha_simple_body(const ShaArgs &a, const uint8_t *suffix) {
    uint64_t t;
    if (!sha_slot(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, t)) return;
    uint32_t id; ChunkRef c;
    const uint8_t *p = sha_chunk(a, t, id, c);
    Sha256State s;
    sha_init(s);
    uint32_t nblk = c.len >> 6;
    for (uint32_t b = 0; b < nblk; b++) {
        uint32_t w[16];
        load_block_be(p + (uint64_t)b * 64, w);
        sha_compress(s, w);
    }
    sha_done<KEYED>(a, suffix, s, p + (uint64_t)nblk * 64, c, id);
}
__global__ void __launch_bounds__(64) k_sha_simple(ShaArgs a) { sha_simple_body<false>(a, nullptr); }
__global__ void __launch_bounds__(64) k_sha_simple_keyed(ShaArgs a, const uint8_t *suffix) { sha_simple_body<true>(a, suffix); }

cudaError_t launch_sha_simple(const ShaArgs &a, cudaStream_t st, const uint8_t *suffix) {
    if (a.chunk_cap == 0) return cudaSuccess;
    uint64_t blocks = (a.chunk_cap + 63) / 64;
    if (suffix) k_sha_simple_keyed<<<(unsigned)blocks, 64, 0, st>>>(a, suffix);
    else k_sha_simple<<<(unsigned)blocks, 64, 0, st>>>(a);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Pipe balancing: the SM's integer work splits over the ALU pipe (LOP3/SHF/PRMT/IADD3) and the FMA pipe (IMAD), 64
// lanes/clk/SM each.  ptxas puts almost all of SHA-256 on the ALU pipe.  Multiplying by constants the compiler cannot
// see (kernel arguments 1, 2^29, 2^22) forces the two logical shifts of the message schedule (mul.hi by 2^(32-n)) and,
// where asked for, the additions (a*1+b) onto IMAD / IMAD.HI.  The throughput kernel moves the shifts only; the split
// kernel's producer moves the shifts and every addition.  tools/sha_lab.cu times other mixes.
// ---------------------------------------------------------------------------
struct Opq { uint32_t one, p29, p22; };

__device__ __forceinline__ uint32_t fma_add(uint32_t a, uint32_t b, const Opq &o) {
    uint32_t d; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(o.one), "r"(b)); return d;
}
__device__ __forceinline__ uint32_t fma_shr3(uint32_t x, const Opq &o) {
    uint32_t d; asm("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(o.p29)); return d;
}
__device__ __forceinline__ uint32_t fma_shr10(uint32_t x, const Opq &o) {
    uint32_t d; asm("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(x), "r"(o.p22)); return d;
}

// Message schedule step of round i on the 16-word ring w (FIPS 180-4 6.2.2 step 1), shifts and additions on the FMA
// pipe: expands W[i] in place when i >= 16 and returns W[i] + K[i].
__device__ __forceinline__ uint32_t sched(uint32_t (&w)[16], int i, const Opq &o) {
    constexpr uint32_t K[64] = {K256_LIST};
    if (i >= 16) {
        uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
        uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ fma_shr3(w15, o);
        uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ fma_shr10(w2, o);
        w[i & 15] = fma_add(fma_add(w[i & 15], s0, o), fma_add(w[(i + 9) & 15], s1, o), o);
    }
    return fma_add(w[i & 15], K[i], o);
}

// sha_compress with the schedule's shifts on the FMA pipe
__device__ __forceinline__ void sha_compress_t(Sha256State &s, uint32_t (&w)[16], const Opq &o) {
    constexpr uint32_t K[64] = {K256_LIST};
    uint32_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        // the schedule stays inline: sched() puts W+K ahead of S1/ch, and ptxas then picks another pipe mix for this loop
        if (i >= 16) {
            uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ fma_shr3(w15, o);
            uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ fma_shr10(w2, o);
            w[i & 15] = (w[i & 15] + s0) + (w[(i + 9) & 15] + s1);
        }
        uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
        uint32_t ch = (e & f) ^ (~e & g);
        uint32_t kw = w[i & 15] + K[i];
        uint32_t t1 = (h + kw) + (S1 + ch);
        uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
        uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t t2 = S0 + mj;
        h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}

// Tuned kernel.  Same one-lane-per-chunk mapping, but BlockStream's loads and the pipe-balanced compression above.
// KEYED: encrypt mode's digest SHA-256(chunk || suffix); the plain instantiation ignores `suffix`
template <bool KEYED>
__global__ void __launch_bounds__(32) k_sha_tuned(ShaArgs a, Opq o, const uint8_t *suffix) {
    uint64_t t;
    if (!sha_slot(a, (uint64_t)blockIdx.x * 32 + threadIdx.x, t)) return;
    uint32_t id; ChunkRef c;
    const uint8_t *p = sha_chunk(a, t, id, c);
    Sha256State s;
    sha_init(s);
    const uint32_t nblk = c.len >> 6;
    BlockStream in(p, nblk);
    for (uint32_t b = 0; b < nblk; b++) {
        uint32_t w[16];
        in.next(b, w);
        sha_compress_t(s, w, o);
    }
    sha_done<KEYED>(a, suffix, s, p + (uint64_t)nblk * 64, c, id);
}

// ---------------------------------------------------------------------------
// Split kernel (default): the per-chunk SHA-256 chain is serial, so the batch's makespan
// is bounded below by the LONGEST chunk (16 MiB) run by ONE lane.  A lone warp is limited
// by its own dependent-issue rate (ALU instructions occupy the 16-lane pipe 2 clk each and
// ncu shows ~0.38 IPC, stall reason "wait"), so the fewer instructions sit on the serial
// chain the faster the tail.  Each CTA = 2 warps over the same 32 chunks, on different SM
// sub-partitions (own ALU/FMA pipes each):
//   warp 0 (producer): LDG.128 loads + prefetch, realign/byte-swap, message schedule,
//                      W[i]+K[i]  -> shared-memory ring (STS.128, conflict free)
//   warp 1 (consumer): only the 64 rounds (10 ALU + 7 FMA instructions per round),
//                      reads W+K with LDS.128
// hand-off through mbarriers (full/empty per stage, 32 arrivals each).  Total work is the
// same as the single-warp kernel; the serial chain per block shrinks from ~1900 to ~1100
// instructions.
// ---------------------------------------------------------------------------
constexpr int SPLIT_STAGES = 3;

// consumer: 64 rounds with W+K supplied, in IADD3 forms (fewest instructions)
__device__ __forceinline__ void sha_rounds(Sha256State &s, const uint4 (&kwv)[16]) {
    uint32_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        const uint4 v = kwv[i >> 2];
        const uint32_t kw = (i & 3) == 0 ? v.x : (i & 3) == 1 ? v.y : (i & 3) == 2 ? v.z : v.w;
        uint32_t hk = h + kw;                     // off the critical path (h is 3 rounds old)
        uint32_t dhk = d + hk;
        uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
        uint32_t ch = (e & f) ^ (~e & g);
        uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
        uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t en = S1 + ch + dhk;              // IADD3
        uint32_t x = S0 + mj + hk;                // IADD3
        uint32_t an = x + S1 + ch;                // IADD3
        h = g; g = f; f = e; e = en; d = c; c = b; b = a; a = an;
    }
    s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}

template <bool KEYED>
__global__ void __launch_bounds__(64) k_sha_split(ShaArgs a, Opq o, const uint8_t *suffix) {
    __shared__ __align__(16) uint4 ring[SPLIT_STAGES][16][32];   // [stage][4 rounds][lane] = W+K
    __shared__ __align__(8) uint64_t bars[2 * SPLIT_STAGES];
    uint64_t t0;
    if (!sha_slot(a, (uint64_t)blockIdx.x * 32, t0)) return;    // whole CTA idle (uniform)
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t t;
    const bool active = sha_slot(a, (uint64_t)blockIdx.x * 32 + lane, t);
    uint32_t id = 0;
    ChunkRef c; c.stream = 0; c.len = 0; c.start = 0;
    const uint8_t *p = a.base;
    if (active) p = sha_chunk(a, t, id, c);
    if (a.arena && active) p = a.arena + a.arena_off[t] + ((uintptr_t)p & 15);   // the gathered copy (same alignment mod 16)
    const uint32_t nblk = c.len >> 6;
    const uint32_t nblk_max = __reduce_max_sync(0xffffffffu, nblk);
    uint32_t full[SPLIT_STAGES], empty[SPLIT_STAGES];
#pragma unroll
    for (int k = 0; k < SPLIT_STAGES; k++) { full[k] = smem_u32(&bars[k]); empty[k] = smem_u32(&bars[SPLIT_STAGES + k]); }
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < SPLIT_STAGES; k++) { mbar_init(full[k], 32); mbar_init(empty[k], 32); }
        mbar_init_fence();
    }
    __syncthreads();

    if (warp == 0) {
        // ------------------------------ producer ------------------------------
        BlockStream in(p, nblk);
        uint32_t stage = 0, phase = 0;
        for (uint32_t b = 0; b < nblk_max; b++) {
            mbar_wait(empty[stage], phase ^ 1);
            if (b < nblk) {
                uint32_t w[16], kw[4];
                in.next(b, w);
#pragma unroll
                for (int i = 0; i < 64; i++) {
                    kw[i & 3] = sched(w, i, o);
                    if ((i & 3) == 3) ring[stage][i >> 2][lane] = make_uint4(kw[0], kw[1], kw[2], kw[3]);
                }
            }
            mbar_arrive(full[stage]);
            if (++stage == SPLIT_STAGES) { stage = 0; phase ^= 1; }
        }
    } else {
        // ------------------------------ consumer ------------------------------
        Sha256State s;
        sha_init(s);
        uint32_t stage = 0, phase = 0;
        for (uint32_t b = 0; b < nblk_max; b++) {
            mbar_wait(full[stage], phase);
            if (b < nblk) {
                uint4 kwv[16];
#pragma unroll
                for (int k = 0; k < 16; k++) kwv[k] = ring[stage][k][lane];
                sha_rounds(s, kwv);
            }
            mbar_arrive(empty[stage]);
            if (++stage == SPLIT_STAGES) { stage = 0; phase ^= 1; }
        }
        if (active) sha_done<KEYED>(a, suffix, s, p + (uint64_t)nblk * 64, c, id);
    }
}

// throughput kernel
cudaError_t launch_sha_tuned(const ShaArgs &a, cudaStream_t st, const uint8_t *suffix) {
    if (a.chunk_cap == 0) return cudaSuccess;
    Opq o{1u, 1u << 29, 1u << 22};
    unsigned blocks = (unsigned)((a.chunk_cap + 31) / 32);
    if (suffix) k_sha_tuned<true><<<blocks, 32, 0, st>>>(a, o, suffix);
    else k_sha_tuned<false><<<blocks, 32, 0, st>>>(a, o, nullptr);
    return cudaGetLastError();
}

// latency kernel (producer/consumer warps).
// When it is launched next to a kernel that already occupies every SM, the CTA scheduler packs its
// few CTAs onto a handful of SMs, where they run several times slower than on an empty GPU.  In the hybrid launch
// (part 1) each CTA therefore also asks for `spread_kb` KiB of dummy dynamic shared memory, which caps the
// CTAs per SM (30 -> 4, 85 -> 2, 112 -> 1) and forces the spread; the throughput kernel uses no shared
// memory and still co-resides.
cudaError_t launch_sha_split(const ShaArgs &a, int spread_kb, cudaStream_t st, const uint8_t *suffix) {
    if (a.chunk_cap == 0) return cudaSuccess;
    Opq o{1u, 1u << 29, 1u << 22};
    unsigned blocks = (unsigned)((a.chunk_cap + 31) / 32);
    size_t dyn = 0;
    if (a.part == 1 && spread_kb > 0) {
        dyn = (size_t)spread_kb * 1024;
        cudaError_t e = cudaFuncSetAttribute(suffix ? k_sha_split<true> : k_sha_split<false>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
        if (e != cudaSuccess) return e;
    }
    if (suffix) k_sha_split<true><<<blocks, 64, dyn, st>>>(a, o, suffix);
    else k_sha_split<false><<<blocks, 64, dyn, st>>>(a, o, nullptr);
    return cudaGetLastError();
}

// number of leading entries (lengths sorted descending) longer than `threshold`, rounded up to 32 and
// capped at `max_head`: the latency partition is small, so when most chunks are long (zero-filled or
// otherwise structured data cuts every chunk at max) only the longest ones go there and the rest stays
// with the throughput kernel on the big partition
__global__ void k_split_point(const uint32_t *len_sorted_desc, const unsigned long long *n_chunks, uint64_t cap,
                              uint32_t threshold, unsigned long long max_head, unsigned long long *n_head) {
    const unsigned long long n = live_count(*n_chunks, cap);
    unsigned long long lo = 0, hi = n;      // first index with len <= threshold (lengths sorted descending)
    while (lo < hi) {
        unsigned long long mid = (lo + hi) >> 1;
        if (len_sorted_desc[mid] > threshold) lo = mid + 1; else hi = mid;
    }
    unsigned long long h = (lo + 31) & ~31ull;
    if (h > max_head) h = max_head & ~31ull;
    if (h > n) h = n;
    *n_head = h;
}
cudaError_t launch_split_point(const uint32_t *len_sorted_desc, const unsigned long long *n_chunks, uint64_t cap,
                               uint32_t threshold, unsigned long long max_head, unsigned long long *n_head, cudaStream_t st) {
    k_split_point<<<1, 1, 0, st>>>(len_sorted_desc, n_chunks, cap, threshold, max_head, n_head);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// Long-chunk arena.  A batch's input buffer is needed until the LAST of its chunks is hashed, and the serial chain of a
// 16 MiB chunk takes ~0.3 s -- ten times longer than everything else of a 16 GiB batch.  With an arena the head chunks
// (the ~11 % of the bytes that take the latency kernel) are copied aside first, the latency kernel reads the copy, and
// the caller gets its buffer back as soon as the bulk pass and this copy are done.
// Placement: slot t starts 128 B aligned and keeps the source's misalignment mod 16, so the gather is a plain uint4 copy
// of the 16-byte vectors a hash of the chunk reads (BlockStream::first_vec / vec_count).
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint64_t arena_slot_bytes(const uint8_t *p, uint32_t len) {
    return (BlockStream::vec_span(p, len) + 127) & ~127ull;
}
__global__ void __launch_bounds__(1024) k_arena_plan(ShaArgs a, unsigned long long *n_head, uint64_t arena_cap, uint64_t *arena_off) {
    __shared__ uint64_t warp_sum[32];
    __shared__ uint64_t carry_s;
    __shared__ unsigned long long fit_s;
    const unsigned long long head = live_count(*n_head, live_count(*a.n_chunks, a.chunk_cap));
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry_s = 0; fit_s = head; }
    __syncthreads();
    for (unsigned long long t0 = 0; t0 < head; t0 += 1024) {
        const unsigned long long t = t0 + threadIdx.x;
        uint64_t need = 0;
        if (t < head) {
            uint32_t id; ChunkRef c;
            need = arena_slot_bytes(sha_chunk(a, t, id, c), c.len);
        }
        uint64_t v = need;   // inclusive scan over the block
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint64_t u = __shfl_up_sync(0xffffffffu, v, d); if (lane >= (uint32_t)d) v += u; }
        if (lane == 31) warp_sum[warp] = v;
        const uint64_t carry = carry_s;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = warp_sum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint64_t u = __shfl_up_sync(0xffffffffu, w, d); if (lane >= (uint32_t)d) w += u; }
            warp_sum[lane] = w;
        }
        __syncthreads();
        const uint64_t incl = carry + v + (warp ? warp_sum[warp - 1] : 0);
        if (t < head) {
            if (incl <= arena_cap) arena_off[t] = incl - need;
            else atomicMin(&fit_s, t);
        }
        if (threadIdx.x == 1023) carry_s = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0 && fit_s < head) *n_head = fit_s & ~31ull;   // whole latency CTAs; the rest stays with the throughput kernel
}
cudaError_t launch_arena_plan(const ShaArgs &a, unsigned long long *n_head, uint64_t arena_cap, uint64_t *arena_off,
                              cudaStream_t st) {
    k_arena_plan<<<1, 1024, 0, st>>>(a, n_head, arena_cap, arena_off);
    return cudaGetLastError();
}
__global__ void __launch_bounds__(256) k_arena_gather(ShaArgs a, uint8_t *arena, const uint64_t *arena_off) {
    const unsigned long long head = live_count(*a.n_head, live_count(*a.n_chunks, a.chunk_cap));
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (unsigned long long t = 0; t < head; t++) {
        uint32_t id; ChunkRef c;
        const uint8_t *p = sha_chunk(a, t, id, c);
        const uint4 *src = BlockStream::first_vec(p);
        uint4 *dst = (uint4 *)(arena + arena_off[t]);
        const uint64_t nvec = BlockStream::vec_count(p, c.len);
        uint64_t v = tid;
        for (; v + 3 * stride < nvec; v += 4 * stride) {
            const uint4 x0 = __ldcs(src + v), x1 = __ldcs(src + v + stride), x2 = __ldcs(src + v + 2 * stride), x3 = __ldcs(src + v + 3 * stride);
            dst[v] = x0; dst[v + stride] = x1; dst[v + 2 * stride] = x2; dst[v + 3 * stride] = x3;
        }
        for (; v < nvec; v += stride) dst[v] = __ldcs(src + v);
    }
}
cudaError_t launch_arena_gather(const ShaArgs &a, uint8_t *arena, const uint64_t *arena_off, int sms, cudaStream_t st) {
    if (a.chunk_cap == 0) return cudaSuccess;
    k_arena_gather<<<(unsigned)(sms > 0 ? sms : 132) * 4, 256, 0, st>>>(a, arena, arena_off);
    return cudaGetLastError();
}

// keys for the longest-first ordering: key = len (sorted descending), val = chunk id.
// Entries past n_chunks get key 0 so they sort last.
__global__ void k_len_keys(const ChunkRef *chunks, const unsigned long long *n_chunks, uint64_t cap, uint32_t *keys,
                           uint32_t *vals) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    unsigned long long n = *n_chunks;
    keys[i] = i < n ? chunks[i].len : 0u;
    vals[i] = (uint32_t)i;
}
cudaError_t launch_len_keys(const ChunkRef *chunks, const unsigned long long *n_chunks, uint64_t cap, uint32_t *keys,
                            uint32_t *vals, cudaStream_t st) {
    if (cap == 0) return cudaSuccess;
    k_len_keys<<<(unsigned)((cap + 255) / 256), 256, 0, st>>>(chunks, n_chunks, cap, keys, vals);
    return cudaGetLastError();
}

// (stream, end_off, digest, flags) records in (stream, chunk) order for the caller
__global__ void k_pack_chunks(const ChunkRef *chunks, const uint8_t *digests, const uint8_t *hit,
                              const unsigned long long *n_chunks, uint64_t cap, pbsgpu_chunk *out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= live_count(*n_chunks, cap)) return;
    ChunkRef c = chunks[i];
    // pbsgpu_chunk = 6 x u64: {stream|flags<<32, end_off, digest[4]}
    uint64_t *o = (uint64_t *)(out + i);
    const uint64_t *d = (const uint64_t *)(digests + i * 32);
    uint32_t flags = (hit && hit[i]) ? PBSGPU_CHUNK_KNOWN : 0u;
    o[0] = (uint64_t)c.stream | ((uint64_t)flags << 32);
    o[1] = c.start + c.len;
    o[2] = d[0]; o[3] = d[1]; o[4] = d[2]; o[5] = d[3];
}
cudaError_t launch_pack_chunks(const ChunkRef *chunks, const uint8_t *digests, const uint8_t *hit,
                               const unsigned long long *n_chunks, uint64_t cap, pbsgpu_chunk *out, cudaStream_t st) {
    if (cap == 0) return cudaSuccess;
    k_pack_chunks<<<(unsigned)((cap + 255) / 256), 256, 0, st>>>(chunks, digests, hit, n_chunks, cap, out);
    return cudaGetLastError();
}

}  // namespace pbsgpu
