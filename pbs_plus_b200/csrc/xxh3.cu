// K7 -- batched XXH3-64 (seed 0, default secret) of n byte ranges: SURVEY.md section 8 "next" row f2.
//
// What it replaces: the per-file content hash of the commit walk -- `h := xxh3.New(); tee := io.TeeReader(f, h);
// ... h.Sum64()` (reference internal/pxarmount/commit.go:717-725) and the second full read of every new file in
// verifyBackedFileHashes (commit.go:957-976).  With the file bytes already in HBM for the chunker, the same
// resident bytes give the xxh3 value: no extra host read.
//
// XXH3's long-input loop is a chain over 1 KiB blocks:  acc <- scramble(acc + S_b)  where S_b[8] is a plain SUM over
// the block's 16 stripes of terms that depend only on the data (acc[i^1] += d_i ; acc[i] += lo32(d_i^k) * hi32(d_i^k)).
// So the work splits into
//   phase A (k_xxh3_blocks, HBM-bound, fully parallel): S_b for every full block -- 4 lanes per block, lane j owns
//           the 16 B column j of each stripe (accumulator pair 2j, 2j+1), 16 independent LDG.128 per lane per block,
//           no cross-lane reduction; 64 B of S written per KiB read;
//   phase B (k_xxh3_chain, latency-bound, tiny): 8 threads per stream (one per accumulator) walk the chain
//           (~8 dependent integer ops per block), then the stream's tail stripes, last stripe, merge and avalanche.
// Streams of <= 1 KiB (all the short-length formulas, and long inputs with no full block) go through k_xxh3_small.
// Scratch for S is bounded: a pass covers blocks [win_lo, win_lo + W) of every stream and the chain state is carried
// between passes, so all streams stay parallel in every pass.
//
// Piece form (pbsgpu_stream_hash_range): each range of a pass starts at its own block index blo[s], and off[s] is the
// position of the range's byte 0 relative to `base` taken modulo 2^64 -- it lies before `base` when the range began in an
// earlier window (only bytes at or after blo[s]'s block, or the tail, are read, and those are in the window or in the
// carry in front of it).  fin[s] says whether the tail is in this pass.  Ranges never overlap, so at most one range is
// unfinished at a window end and carries chain state into the next pass.  That state is read from state[0..8) (by the
// pass's first range, when it began earlier) and written to state_out[0..8) (by its last range, when it goes on): two
// slots, so a pass whose first range reads the carried state while its last range saves its own has no
// read-after-write race between their threads.  The caller swaps the slots between passes.
#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

static const uint8_t XSECRET[192] = {
    0xb8, 0xfe, 0x6c, 0x39, 0x23, 0xa4, 0x4b, 0xbe, 0x7c, 0x01, 0x81, 0x2c, 0xf7, 0x21, 0xad, 0x1c,
    0xde, 0xd4, 0x6d, 0xe9, 0x83, 0x90, 0x97, 0xdb, 0x72, 0x40, 0xa4, 0xa4, 0xb7, 0xb3, 0x67, 0x1f,
    0xcb, 0x79, 0xe6, 0x4e, 0xcc, 0xc0, 0xe5, 0x78, 0x82, 0x5a, 0xd0, 0x7d, 0xcc, 0xff, 0x72, 0x21,
    0xb8, 0x08, 0x46, 0x74, 0xf7, 0x43, 0x24, 0x8e, 0xe0, 0x35, 0x90, 0xe6, 0x81, 0x3a, 0x26, 0x4c,
    0x3c, 0x28, 0x52, 0xbb, 0x91, 0xc3, 0x00, 0xcb, 0x88, 0xd0, 0x65, 0x8b, 0x1b, 0x53, 0x2e, 0xa3,
    0x71, 0x64, 0x48, 0x97, 0xa2, 0x0d, 0xf9, 0x4e, 0x38, 0x19, 0xef, 0x46, 0xa9, 0xde, 0xac, 0xd8,
    0xa8, 0xfa, 0x76, 0x3f, 0xe3, 0x9c, 0x34, 0x3f, 0xf9, 0xdc, 0xbb, 0xc7, 0xc7, 0x0b, 0x4f, 0x1d,
    0x8a, 0x51, 0xe0, 0x4b, 0xcd, 0xb4, 0x59, 0x31, 0xc8, 0x9f, 0x7e, 0xc9, 0xd9, 0x78, 0x73, 0x64,
    0xea, 0xc5, 0xac, 0x83, 0x34, 0xd3, 0xeb, 0xc3, 0xc5, 0x81, 0xa0, 0xff, 0xfa, 0x13, 0x63, 0xeb,
    0x17, 0x0d, 0xdd, 0x51, 0xb7, 0xf0, 0xda, 0x49, 0xd3, 0x16, 0x55, 0x26, 0x29, 0xd4, 0x68, 0x9e,
    0x2b, 0x16, 0xbe, 0x58, 0x7d, 0x47, 0xa1, 0xfc, 0x8f, 0xf8, 0xb8, 0xd1, 0x7a, 0xd0, 0x31, 0xce,
    0x45, 0xcb, 0x3a, 0x8f, 0x95, 0x16, 0x04, 0x28, 0xaf, 0xd7, 0xfb, 0xca, 0xbb, 0x4b, 0x40, 0x7e,
};

// Device table: [0, 184) = the 23 aligned words sec64(8 t), t = 0..22 (phase A) ; [192, 384) = the secret bytes.
constexpr int XT_WORDS = 24;
constexpr int XT_BYTES = XT_WORDS * 8 + 192;
size_t xxh3_tables_bytes() { return XT_BYTES; }
void xxh3_fill_tables_host(void *dst) {
    uint8_t *p = (uint8_t *)dst;
    memset(p, 0, XT_BYTES);
    memcpy(p, XSECRET, 184);            // little-endian words sec64(8 t) are just the bytes themselves
    memcpy(p + XT_WORDS * 8, XSECRET, 192);
}
uint64_t xxh3_block_bytes() { return 1024; }

constexpr uint32_t XP32_1 = 0x9E3779B1u, XP32_2 = 0x85EBCA77u, XP32_3 = 0xC2B2AE3Du;
constexpr uint64_t XP64_1 = 0x9E3779B185EBCA87ull, XP64_2 = 0xC2B2AE3D27D4EB4Full, XP64_3 = 0x165667B19E3779F9ull,
                   XP64_4 = 0x85EBCA77C2B2AE63ull, XP64_5 = 0x27D4EB2F165667C5ull, XPMX1 = 0x165667919E3779F9ull,
                   XPMX2 = 0x9FB21C651E98DF25ull;

__device__ __forceinline__ uint64_t ld64u(const uint8_t *p) {   // unaligned little-endian load (tails only)
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i);
    return v;
}
__device__ __forceinline__ uint32_t ld32u(const uint8_t *p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t mul32x32(uint64_t k) { return (uint64_t)(uint32_t)k * (uint64_t)(uint32_t)(k >> 32); }
__device__ __forceinline__ uint64_t fold128(uint64_t a, uint64_t b) { return (a * b) ^ __umul64hi(a, b); }
__device__ __forceinline__ uint64_t aval3(uint64_t h) { h ^= h >> 37; h *= XPMX1; h ^= h >> 32; return h; }
__device__ __forceinline__ uint64_t aval64(uint64_t h) { h ^= h >> 33; h *= XP64_2; h ^= h >> 29; h *= XP64_3; h ^= h >> 32; return h; }
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
    return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | __byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}
__device__ __forceinline__ uint64_t mix16(const uint8_t *in, const uint8_t *sec) {
    return fold128(ld64u(in) ^ ld64u(sec), ld64u(in + 8) ^ ld64u(sec + 8));
}
__device__ __forceinline__ uint64_t acc_init(int i) {
    switch (i) {
        case 0: return XP32_3; case 1: return XP64_1; case 2: return XP64_2; case 3: return XP64_3;
        case 4: return XP64_4; case 5: return XP32_2; case 6: return XP64_5; default: return XP32_1;
    }
}
// full 1 KiB blocks of a stream (they are followed by a scramble): (len - 1) / 1024 for long inputs
__device__ __forceinline__ uint64_t full_blocks(uint64_t len) { return len > 240 ? (len - 1) >> 10 : 0; }

struct XxhArgs {
    const uint8_t *base;
    const uint64_t *off, *len;
    const uint64_t *first;   // [n + 1] prefix of the blocks each stream has in this pass
    uint32_t n;
    uint64_t total;          // blocks in this pass
    uint64_t win_lo, win;    // the pass covers per-stream blocks [win_lo, win_lo + win)
    const uint8_t *tab;      // xxh3_fill_tables_host image
    uint64_t *S;             // [total][8]
    uint64_t *state;         // [n][8] chain state between passes
    uint64_t *out;           // [n]
    const uint64_t *blo;     // piece form: [n] first block of the range in this pass (NULL: win_lo for every stream)
    const uint8_t *fin;      // piece form: [n] the range ends in this pass
    uint64_t *state_out;     // piece form: [8] chain state of the range that goes on after this pass
};

constexpr int XA_U = 8;   // blocks per 4-lane group (8 KiB): one stream search per group

// ---- phase A ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_xxh3_blocks(XxhArgs a) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t j = (uint32_t)tid & 3;
    const uint64_t g0 = (tid >> 2) * XA_U;
    if (g0 >= a.total) return;
    uint64_t K[17];   // K[t] = sec64(8 (2 j + t))
    const uint64_t *kw = (const uint64_t *)a.tab + 2 * j;
#pragma unroll
    for (int t = 0; t < 17; t++) K[t] = __ldg(kw + t);
    uint32_t s = owner_of(a.first, a.n, g0);
    uint64_t s_first = a.first[s], s_next = a.first[s + 1];
#pragma unroll 1
    for (int u = 0; u < XA_U; u++) {
        const uint64_t g = g0 + u;
        if (g >= a.total) break;
        while (g >= s_next) { s++; s_first = s_next; s_next = a.first[s + 1]; }
        const uint64_t lo = a.blo ? a.blo[s] : a.win_lo;
        const uint8_t *p = a.base + (a.off[s] + ((lo + (g - s_first)) << 10) + j * 16);
        uint64_t a0 = 0, a1 = 0;
        if ((((uintptr_t)p) & 15) == 0) {
            ulonglong2 d[16];
#pragma unroll
            for (int st = 0; st < 16; st++) d[st] = *(const ulonglong2 *)(p + st * 64);
#pragma unroll
            for (int st = 0; st < 16; st++) {
                a0 += d[st].y + mul32x32(d[st].x ^ K[st]);
                a1 += d[st].x + mul32x32(d[st].y ^ K[st + 1]);
            }
        } else {   // stream not 16 B aligned in memory: same arithmetic from byte loads (slow, rare)
#pragma unroll 1
            for (int st = 0; st < 16; st++) {
                const uint64_t x = ld64u(p + st * 64), y = ld64u(p + st * 64 + 8);
                a0 += y + mul32x32(x ^ __ldg(kw + st));       // K[] stays in registers: no dynamic index here
                a1 += x + mul32x32(y ^ __ldg(kw + st + 1));
            }
        }
        *(ulonglong2 *)(a.S + g * 8 + 2 * j) = make_ulonglong2(a0, a1);
    }
}

// ---- phase B ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t stripe_term(const uint8_t *in, const uint8_t *sec, int i) {
    return ld64u(in + 8 * (i ^ 1)) + mul32x32(ld64u(in + 8 * i) ^ ld64u(sec + 8 * i));
}

__global__ void __launch_bounds__(256) k_xxh3_chain(XxhArgs a) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t i = (uint32_t)tid & 7, lane = threadIdx.x & 31;
    const uint64_t sidx = tid >> 3;
    const bool in_range = sidx < a.n;
    const uint32_t s = in_range ? (uint32_t)sidx : 0;
    const uint64_t len = in_range ? a.len[s] : 0;
    const uint64_t nb = full_blocks(len);
    uint64_t lo, hi;
    bool active, last;
    if (a.blo) {   // piece form: a range may have no block in the pass and only its tail
        lo = in_range ? a.blo[s] : 0;
        hi = in_range ? lo + (a.first[s + 1] - a.first[s]) : 0;
        last = in_range && nb != 0 && a.fin[s];
        active = in_range && (lo < hi || last);
    } else {
        lo = nb < a.win_lo ? nb : a.win_lo;
        hi = nb < a.win_lo + a.win ? nb : a.win_lo + a.win;
        active = in_range && lo < hi;
        last = active && hi == nb;
    }
    const uint8_t *sec = a.tab + XT_WORDS * 8;
    const uint64_t *state_in = a.state + (a.blo ? 0 : (uint64_t)s * 8) + i;
    uint64_t *state_out = (a.blo ? a.state_out : a.state + (uint64_t)s * 8) + i;
    uint64_t acc = 0;
    if (active) {
        acc = lo == 0 ? acc_init(i) : *state_in;
        const uint64_t ks = ld64u(sec + 128 + 8 * i);
        const uint64_t *sp = a.S + a.first[s] * 8 + i;
        // The loads do not depend on the chain: keep the next 16 block sums in flight while the current 16 are
        // consumed, so the ~30-cycle dependent step (add, shift, xor, 64x32 multiply) is all that is left per block.
        constexpr int PB = 16;
        const uint64_t cnt = hi - lo;
        uint64_t cur[PB], nxt[PB];
#pragma unroll
        for (int k = 0; k < PB; k++) cur[k] = (uint64_t)k < cnt ? sp[(uint64_t)k * 8] : 0;
        for (uint64_t b = 0; b < cnt; b += PB) {
            if (b + 2 * PB <= cnt) {
#pragma unroll
                for (int k = 0; k < PB; k++) nxt[k] = sp[(b + PB + k) * 8];
            } else {
#pragma unroll
                for (int k = 0; k < PB; k++) nxt[k] = b + PB + k < cnt ? sp[(b + PB + k) * 8] : 0;
            }
            if (b + PB <= cnt) {
#pragma unroll
                for (int k = 0; k < PB; k++) { acc += cur[k]; acc = (acc ^ (acc >> 47) ^ ks) * XP32_1; }
            } else {
#pragma unroll
                for (int k = 0; k < PB; k++)
                    if (b + k < cnt) { acc += cur[k]; acc = (acc ^ (acc >> 47) ^ ks) * XP32_1; }
            }
#pragma unroll
            for (int k = 0; k < PB; k++) cur[k] = nxt[k];
        }
        if (!last) *state_out = acc;
        else {
            const uint64_t d = a.off[s];
            const uint64_t ns = ((len - 1) - (nb << 10)) >> 6;
            for (uint64_t st = 0; st < ns; st++) acc += stripe_term(a.base + (d + (nb << 10) + 64 * st), sec + 8 * st, i);
            acc += stripe_term(a.base + (d + len - 64), sec + 192 - 64 - 7, i);
        }
    }
    // merge: accumulators of one stream sit in 8 consecutive lanes
    uint64_t r = len * XP64_1;
    const uint32_t gbase = lane & ~7u;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint64_t x = __shfl_sync(0xffffffffu, acc, gbase + 2 * k), y = __shfl_sync(0xffffffffu, acc, gbase + 2 * k + 1);
        r += fold128(x ^ ld64u(sec + 11 + 16 * k), y ^ ld64u(sec + 11 + 16 * k + 8));
    }
    if (last && i == 0) a.out[s] = aval3(r);
}

// ---- short inputs and long inputs without a full block (len <= 1024): one thread per stream ------------------------
__global__ void __launch_bounds__(128) k_xxh3_small(XxhArgs a) {
    const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= a.n) return;
    const uint32_t s = (uint32_t)tid;
    const uint64_t len = a.len[s];
    if (full_blocks(len) != 0) return;
    const uint8_t *in = a.base + (int64_t)a.off[s];   // piece form: a carried range starts in front of `base`
    const uint8_t *S = a.tab + XT_WORDS * 8;
    uint64_t h;
    if (len == 0) h = aval64(ld64u(S + 56) ^ ld64u(S + 64));
    else if (len <= 3) {
        const uint32_t comb = ((uint32_t)in[0] << 16) | ((uint32_t)in[len >> 1] << 24) | in[len - 1] | ((uint32_t)len << 8);
        h = aval64((uint64_t)comb ^ (uint64_t)(ld32u(S) ^ ld32u(S + 4)));
    } else if (len <= 8) {
        h = ((uint64_t)ld32u(in + len - 4) + ((uint64_t)ld32u(in) << 32)) ^ (ld64u(S + 8) ^ ld64u(S + 16));
        h ^= rotl64(h, 49) ^ rotl64(h, 24); h *= XPMX2; h ^= (h >> 35) + len; h *= XPMX2;
        h ^= h >> 28;
    } else if (len <= 16) {
        const uint64_t lo = ld64u(in) ^ (ld64u(S + 24) ^ ld64u(S + 32)), hi = ld64u(in + len - 8) ^ (ld64u(S + 40) ^ ld64u(S + 48));
        h = aval3(len + bswap64(lo) + hi + fold128(lo, hi));
    } else if (len <= 128) {
        uint64_t acc = len * XP64_1;
        for (int k = (int)((len - 1) / 32); k >= 0; k--) {
            acc += mix16(in + 16 * k, S + 32 * k);
            acc += mix16(in + len - 16 * (k + 1), S + 32 * k + 16);
        }
        h = aval3(acc);
    } else if (len <= 240) {
        uint64_t acc = len * XP64_1;
        for (int k = 0; k < 8; k++) acc += mix16(in + 16 * k, S + 16 * k);
        uint64_t end = mix16(in + len - 16, S + 136 - 17);
        acc = aval3(acc);
        for (uint32_t k = 8; k < len / 16; k++) end += mix16(in + 16 * k, S + 16 * (k - 8) + 3);
        h = aval3(acc + end);
    } else {   // 241..1024: no full block; tail stripes, last stripe, merge
        uint64_t acc[8];
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] = acc_init(k);
        const uint64_t ns = (len - 1) >> 6;
        for (uint64_t st = 0; st < ns; st++) {
#pragma unroll
            for (int k = 0; k < 8; k++) acc[k] += stripe_term(in + 64 * st, S + 8 * st, k);
        }
#pragma unroll
        for (int k = 0; k < 8; k++) acc[k] += stripe_term(in + len - 64, S + 192 - 64 - 7, k);
        uint64_t r = len * XP64_1;
#pragma unroll
        for (int k = 0; k < 4; k++) r += fold128(acc[2 * k] ^ ld64u(S + 11 + 16 * k), acc[2 * k + 1] ^ ld64u(S + 11 + 16 * k + 8));
        h = aval3(r);
    }
    a.out[s] = h;
}

// One pass: S for the pass's blocks, then the chain over them (finalising streams whose last block is in the pass).
cudaError_t launch_xxh3_pass(const uint8_t *base, const uint64_t *off, const uint64_t *len, const uint64_t *first, uint32_t n,
                             uint64_t total, uint64_t win_lo, uint64_t win, const void *tab, uint64_t *S, uint64_t *state,
                             uint64_t *out, cudaStream_t st) {
    XxhArgs a{base, off, len, first, n, total, win_lo, win, (const uint8_t *)tab, S, state, out, nullptr, nullptr, nullptr};
    if (total) {
        const uint64_t groups = (total + XA_U - 1) / XA_U, threads = groups * 4;
        k_xxh3_blocks<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        k_xxh3_chain<<<(unsigned)(((uint64_t)n * 8 + 255) / 256), 256, 0, st>>>(a);
        return cudaGetLastError();
    }
    return cudaSuccess;
}

cudaError_t launch_xxh3_small(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint32_t n, const void *tab,
                              uint64_t *out, cudaStream_t st) {
    XxhArgs a{base, off, len, nullptr, n, 0, 0, 0, (const uint8_t *)tab, nullptr, nullptr, out, nullptr, nullptr, nullptr};
    k_xxh3_small<<<(n + 127) / 128, 128, 0, st>>>(a);
    return cudaGetLastError();
}

// Piece form: the ranges' blocks in this pass (prefix `first`, from block blo[s]), the chain carried in from state_in[0..8)
// and out to state_out[0..8) (distinct slots), and the finish of every range with fin[s] -- long ranges in the chain
// kernel, ranges of <= 1 KiB in k_xxh3_small.
cudaError_t launch_xxh3_pieces(const uint8_t *base, const uint64_t *off, const uint64_t *len, const uint64_t *first,
                               const uint64_t *blo, const uint8_t *fin, uint32_t n, uint64_t total, const void *tab,
                               uint64_t *S, uint64_t *state_in, uint64_t *state_out, uint64_t *out, cudaStream_t st) {
    XxhArgs a{base, off, len, first, n, total, 0, 0, (const uint8_t *)tab, S, state_in, out, blo, fin, state_out};
    if (n == 0) return cudaSuccess;
    if (total) {
        const uint64_t groups = (total + XA_U - 1) / XA_U, threads = groups * 4;
        k_xxh3_blocks<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    k_xxh3_chain<<<(unsigned)(((uint64_t)n * 8 + 255) / 256), 256, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_xxh3_small<<<(n + 127) / 128, 128, 0, st>>>(a);
    return cudaGetLastError();
}

// XXH3-64 of the empty input (a constant of the secret), for empty ranges that no window holds
uint64_t xxh3_empty_host() {
    uint64_t a = 0, b = 0;
    for (int i = 0; i < 8; i++) { a |= (uint64_t)XSECRET[56 + i] << (8 * i); b |= (uint64_t)XSECRET[64 + i] << (8 * i); }
    uint64_t h = a ^ b;
    h ^= h >> 33; h *= XP64_2; h ^= h >> 29; h *= XP64_3; h ^= h >> 32;
    return h;
}

}  // namespace pbsgpu
