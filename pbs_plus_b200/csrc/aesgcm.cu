// pbs_plus_b200/csrc/aesgcm.cu -- K11: AES-256-GCM of n byte ranges (the payloads of encrypted DataBlobs).
//
// Upstream PBS encrypts a blob's payload (the raw chunk, or its zstd frame when that is smaller) with AES-256-GCM under
// the client key, a 16-byte IV and no AAD (pbs-tools crypt_config.rs, restated; UNVERIFIED-HERE).  A 16-byte IV takes
// GCM's general path: J0 = GHASH_H(IV || 0^64 || [128]_64), keystream block i = E_K(inc32^i(J0)), and
// tag = E_K(J0) ^ GHASH_H(C || [0]_64 || [8 |C|]_64).  J0 and E_K(J0) are a few operations per blob and are computed on
// the host; everything that is proportional to the payload runs here.
//
// Work split.  A message of m 16-byte blocks is cut into segments of GCM_SEG_BLOCKS (16 KiB); one warp owns a segment
// and lane l takes blocks l, l+32, l+64, ... of it, so every load and store of the warp is 512 contiguous bytes.
//  - CTR: each lane encrypts its counter blocks (T-table AES, one table T0 lane-replicated in shared memory as K6 does
//    for its CRC tables: the bank of a lookup is the lane, so the 16 lookups of a round never conflict; T1..T3 are
//    rotations of T0 and the S-box is a byte of T0) and XORs them into the data in place.
//  - GHASH is linear over GF(2^128), so it splits like K6's CRC: lane l runs Horner over its own blocks with the step
//    H^32 (an 8-bit Shoup table of H^32 in shared memory), then scales the result by H^(e - last block of the lane),
//    where e is the segment's last block, and the 32 lanes XOR their results: the segment's GHASH relative to e.
//  - k_gcm_tag (one thread per message) chains the segments by Horner with H^GCM_SEG_BLOCKS (Shoup table), the last
//    one with H^k (k < GCM_SEG_BLOCKS, table of powers), appends the length block and XORs E_K(J0): the tag.
// The counter is inc32: only the low 32-bit word advances, wrapping modulo 2^32 inside a message as GCM specifies.
// Decryption (k_gcm_ctr_ghash<true>) is the same CTR transform; GHASH then runs over the input blocks before the XOR,
// with the partial last block masked first (its granule can hold bytes of the next blob), and k_gcm_tag yields the tag
// the ciphertext should carry, which the caller compares with the blob's.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

// Tables of one key (host copy in pbsgpu_crypt, device copy uploaded once).  GF(2^128) elements are 4 big-endian
// words: word 0 holds bytes 0..3 of the GCM block, the most significant bit of byte 0 is the coefficient of x^0.
struct GcmTables {
    uint32_t rk[60];                      // AES-256 round keys (FIPS-197 word order)
    uint32_t t0[256];                     // T0[x] = {2 S(x), S(x), S(x), 3 S(x)}, most significant byte first
    uint32_t r8[256];                     // reduction of the byte shifted out by a multiplication with x^8
    uint32_t m1[256][4];                  // Shoup table: m1[b] = b * H (b as the polynomial of block byte 0)
    uint32_t m32[256][4];                 // ... of H^32 (lane Horner step)
    uint32_t mseg[256][4];                // ... of H^GCM_SEG_BLOCKS (segment chain step)
    uint32_t hp[GCM_SEG_BLOCKS + 1][4];   // H^0 .. H^GCM_SEG_BLOCKS
};

// ---- GF(2^128), GCM bit order ------------------------------------------------------------------------------------
// z = x * y, bit by bit (the general product: used once per lane and segment, and on the host)
__host__ __device__ inline void gf_mul(const uint32_t x[4], const uint32_t y[4], uint32_t z[4]) {
    uint32_t v0 = y[0], v1 = y[1], v2 = y[2], v3 = y[3], z0 = 0, z1 = 0, z2 = 0, z3 = 0;
    for (int i = 0; i < 128; i++) {
        const uint32_t m = 0u - ((x[i >> 5] >> (31 - (i & 31))) & 1u);
        z0 ^= v0 & m; z1 ^= v1 & m; z2 ^= v2 & m; z3 ^= v3 & m;
        const uint32_t r = 0u - (v3 & 1u);
        v3 = (v3 >> 1) | (v2 << 31); v2 = (v2 >> 1) | (v1 << 31); v1 = (v1 >> 1) | (v0 << 31); v0 = (v0 >> 1) ^ (r & 0xE1000000u);
    }
    z[0] = z0; z[1] = z1; z[2] = z2; z[3] = z3;
}

// z = z * Y with Y's 8-bit Shoup table m[256][4] and the reduction table r8: Horner over the bytes of z from byte 15
// to byte 0, each step a multiplication by x^8 (shift right by 8, reduce the byte shifted out) and one table entry.
template <class M, class R>
__host__ __device__ __forceinline__ void gf_mul_table(uint32_t z[4], M m, R r8) {
    uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
#pragma unroll
    for (int k = 15; k >= 0; k--) {
        const uint32_t rb = r8(a3 & 0xFFu);
        a3 = (a3 >> 8) | (a2 << 24); a2 = (a2 >> 8) | (a1 << 24); a1 = (a1 >> 8) | (a0 << 24); a0 = (a0 >> 8) ^ rb;
        const uint4 t = m((z[k >> 2] >> (24 - 8 * (k & 3))) & 0xFFu);
        a0 ^= t.x; a1 ^= t.y; a2 ^= t.z; a3 ^= t.w;
    }
    z[0] = a0; z[1] = a1; z[2] = a2; z[3] = a3;
}

// ---- host: key schedule and tables ----------------------------------------------------------------------------------
static uint8_t gf8_mul(uint8_t a, uint8_t b) {
    uint8_t p = 0;
    for (int i = 0; i < 8; i++) {
        if (b & 1) p ^= a;
        a = (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1B : 0));
        b >>= 1;
    }
    return p;
}
static void aes_sbox(uint8_t s[256]) {
    for (int x = 0; x < 256; x++) {
        uint8_t inv = 0;   // x^254 = x^-1 in GF(2^8) (0 for 0)
        if (x) { inv = 1; for (int k = 0; k < 254; k++) inv = gf8_mul(inv, (uint8_t)x); }
        uint8_t v = inv;
        for (int r = 1; r < 5; r++) v ^= (uint8_t)((inv << r) | (inv >> (8 - r)));
        s[x] = v ^ 0x63;
    }
}
static inline uint32_t ror32(uint32_t x, int r) { return (x >> r) | (x << (32 - r)); }

static void shoup_table(const uint32_t y[4], uint32_t m[256][4]) {
    for (uint32_t b = 0; b < 256; b++) {
        const uint32_t x[4] = {b << 24, 0, 0, 0};
        gf_mul(x, y, m[b]);
    }
}

void gcm_fill_tables_host(const uint8_t key[32], void *dst) {
    GcmTables *t = (GcmTables *)dst;
    uint8_t s[256];
    aes_sbox(s);
    for (int x = 0; x < 256; x++) {
        const uint8_t a = s[x], a2 = gf8_mul(a, 2), a3 = gf8_mul(a, 3);
        t->t0[x] = (uint32_t)a2 << 24 | (uint32_t)a << 16 | (uint32_t)a << 8 | a3;
    }
    auto sub = [&](uint32_t w) {
        return (uint32_t)s[w >> 24] << 24 | (uint32_t)s[(w >> 16) & 255] << 16 | (uint32_t)s[(w >> 8) & 255] << 8 | s[w & 255];
    };
    for (int i = 0; i < 8; i++) t->rk[i] = (uint32_t)key[4 * i] << 24 | (uint32_t)key[4 * i + 1] << 16 | (uint32_t)key[4 * i + 2] << 8 | key[4 * i + 3];
    uint32_t rcon = 1;
    for (int i = 8; i < 60; i++) {
        uint32_t w = t->rk[i - 1];
        if (i % 8 == 0) { w = sub((w << 8) | (w >> 24)) ^ (rcon << 24); rcon = gf8_mul((uint8_t)rcon, 2); }
        else if (i % 8 == 4) w = sub(w);
        t->rk[i] = t->rk[i - 8] ^ w;
    }
    for (uint32_t b = 0; b < 256; b++) {   // (block with byte 15 = b) * x^8 lands in the top 16 bits
        uint32_t v[4] = {0, 0, 0, b};
        for (int k = 0; k < 8; k++) {
            const uint32_t r = v[3] & 1u;
            v[3] = (v[3] >> 1) | (v[2] << 31); v[2] = (v[2] >> 1) | (v[1] << 31); v[1] = (v[1] >> 1) | (v[0] << 31); v[0] = (v[0] >> 1) ^ (r ? 0xE1000000u : 0u);
        }
        t->r8[b] = v[0];
    }
    uint32_t h[4];
    const uint32_t zero[4] = {0, 0, 0, 0};
    gcm_encrypt_block_host(t, zero, h);    // H = E_K(0^128)
    t->hp[0][0] = 0x80000000u; t->hp[0][1] = t->hp[0][2] = t->hp[0][3] = 0;   // 1
    for (uint32_t k = 1; k <= GCM_SEG_BLOCKS; k++) gf_mul(t->hp[k - 1], h, t->hp[k]);
    shoup_table(t->hp[1], t->m1);
    shoup_table(t->hp[32], t->m32);
    shoup_table(t->hp[GCM_SEG_BLOCKS], t->mseg);
    memset(s, 0, sizeof s);
}

void gcm_encrypt_block_host(const void *tables, const uint32_t in[4], uint32_t out[4]) {
    const GcmTables *t = (const GcmTables *)tables;
    const uint32_t *T = t->t0, *rk = t->rk;
    uint32_t s0 = in[0] ^ rk[0], s1 = in[1] ^ rk[1], s2 = in[2] ^ rk[2], s3 = in[3] ^ rk[3];
    for (int r = 1; r < 14; r++) {
        const uint32_t a = T[s0 >> 24] ^ ror32(T[(s1 >> 16) & 255], 8) ^ ror32(T[(s2 >> 8) & 255], 16) ^ ror32(T[s3 & 255], 24) ^ rk[4 * r];
        const uint32_t b = T[s1 >> 24] ^ ror32(T[(s2 >> 16) & 255], 8) ^ ror32(T[(s3 >> 8) & 255], 16) ^ ror32(T[s0 & 255], 24) ^ rk[4 * r + 1];
        const uint32_t c = T[s2 >> 24] ^ ror32(T[(s3 >> 16) & 255], 8) ^ ror32(T[(s0 >> 8) & 255], 16) ^ ror32(T[s1 & 255], 24) ^ rk[4 * r + 2];
        const uint32_t d = T[s3 >> 24] ^ ror32(T[(s0 >> 16) & 255], 8) ^ ror32(T[(s1 >> 8) & 255], 16) ^ ror32(T[s2 & 255], 24) ^ rk[4 * r + 3];
        s0 = a; s1 = b; s2 = c; s3 = d;
    }
    auto S = [&](uint32_t x) { return (T[x & 255] >> 8) & 255u; };
    out[0] = (S(s0 >> 24) << 24 | S(s1 >> 16) << 16 | S(s2 >> 8) << 8 | S(s3)) ^ rk[56];
    out[1] = (S(s1 >> 24) << 24 | S(s2 >> 16) << 16 | S(s3 >> 8) << 8 | S(s0)) ^ rk[57];
    out[2] = (S(s2 >> 24) << 24 | S(s3 >> 16) << 16 | S(s0 >> 8) << 8 | S(s1)) ^ rk[58];
    out[3] = (S(s3 >> 24) << 24 | S(s0 >> 16) << 16 | S(s1 >> 8) << 8 | S(s2)) ^ rk[59];
}

// J0 of a 16-byte IV: GHASH_H(IV || 0^64 || [128]_64) = (IV * H ^ [128]_128) * H
void gcm_j0_host(const void *tables, const uint8_t iv[16], uint32_t j0[4]) {
    const GcmTables *t = (const GcmTables *)tables;
    uint32_t y[4];
    for (int i = 0; i < 4; i++) y[i] = (uint32_t)iv[4 * i] << 24 | (uint32_t)iv[4 * i + 1] << 16 | (uint32_t)iv[4 * i + 2] << 8 | iv[4 * i + 3];
    gf_mul(y, t->hp[1], j0);
    j0[3] ^= 128u;
    gf_mul(j0, t->hp[1], y);
    for (int i = 0; i < 4; i++) j0[i] = y[i];
}

size_t gcm_tables_bytes() { return sizeof(GcmTables); }

// ---- device -------------------------------------------------------------------------------------------------------
constexpr int GCM_THREADS = 256;
constexpr int GCM_SMEM = 256 * 32 * 4 /*T0 per lane*/ + 256 * 16 /*m32*/ + 256 * 4 /*r8*/ + 60 * 4 /*rk*/;

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }
__device__ __forceinline__ uint32_t rorr(uint32_t x, int r) { return __funnelshift_r(x, x, r); }

// gf_mul with the word loop unrolled, so x is never indexed at run time and stays in registers: gf_mul's x[i >> 5]
// puts x on the stack (the 16-byte frame of the encrypt kernel, whose code is kept as it is)
__device__ __forceinline__ void gf_mul_reg(const uint32_t x[4], const uint32_t y[4], uint32_t z[4]) {
    uint32_t v0 = y[0], v1 = y[1], v2 = y[2], v3 = y[3], z0 = 0, z1 = 0, z2 = 0, z3 = 0;
#pragma unroll
    for (int w = 0; w < 4; w++) {
        const uint32_t xw = x[w];
#pragma unroll 1
        for (int i = 31; i >= 0; i--) {
            const uint32_t m = 0u - ((xw >> i) & 1u);
            z0 ^= v0 & m; z1 ^= v1 & m; z2 ^= v2 & m; z3 ^= v3 & m;
            const uint32_t r = 0u - (v3 & 1u);
            v3 = (v3 >> 1) | (v2 << 31); v2 = (v2 >> 1) | (v1 << 31); v1 = (v1 >> 1) | (v0 << 31); v0 = (v0 >> 1) ^ (r & 0xE1000000u);
        }
    }
    z[0] = z0; z[1] = z1; z[2] = z2; z[3] = z3;
}

// Bytes of a block with r valid bytes (r < 16): keep bytes 0 .. r-1 of the big-endian words
__device__ __forceinline__ uint32_t keep_mask(int r, int word) {
    const int v = r - 4 * word;
    return v >= 4 ? 0xFFFFFFFFu : v <= 0 ? 0u : ~(0xFFFFFFFFu >> (8 * v));
}

// msg[i] covers dev bytes [src, src + len) (any alignment) and writes its CTR transform to dst (16 B aligned, room for
// whole blocks; bytes past len are zero); part[seg] = the segment's GHASH of the ciphertext relative to its last block.
// Encrypting, the ciphertext is the output; decrypting (DECRYPT), it is the input, hashed before the XOR.
template <bool DECRYPT>
__global__ void __launch_bounds__(GCM_THREADS) k_gcm_ctr_ghash(const GcmMsg *msg, const uint64_t *seg_first, uint32_t n,
                                                               uint64_t total_segs, const GcmTables *tab, uint4 *part) {
    extern __shared__ __align__(16) uint8_t gcm_smem[];
    uint32_t *TR = (uint32_t *)gcm_smem;                    // [256][32] T0 per lane
    uint4 *M32 = (uint4 *)(TR + 256 * 32);                  // [256]
    uint32_t *R8 = (uint32_t *)(M32 + 256), *RK = R8 + 256;
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) TR[i] = tab->t0[i >> 5];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        M32[i] = make_uint4(tab->m32[i][0], tab->m32[i][1], tab->m32[i][2], tab->m32[i][3]);
        R8[i] = tab->r8[i];
    }
    if (threadIdx.x < 60) RK[threadIdx.x] = tab->rk[threadIdx.x];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, lane4 = lane << 2;
    const uint8_t *TB = (const uint8_t *)TR;
    // T0[byte of x at bit `sh`] through this lane's replica: byte offset (byte << 7) | lane * 4
#define GT(x, sh) (*(const uint32_t *)(TB + ((((sh) >= 7 ? (x) >> ((sh) - 7) : (x) << (7 - (sh))) & 0x7F80u) | lane4)))
    const uint64_t warps_total = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t g = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < total_segs; g += warps_total) {
        const uint32_t r = owner_of(seg_first, n, g);
        const GcmMsg mm = msg[r];
        const uint64_t seg = g - seg_first[r], m = (mm.len + 15) >> 4, b0 = seg * GCM_SEG_BLOCKS;
        const uint64_t e = (b0 + GCM_SEG_BLOCKS < m ? b0 + GCM_SEG_BLOCKS : m) - 1;   // last block of the segment
        const uint8_t *src = (const uint8_t *)mm.src;
        const uint32_t mis = (uint32_t)(mm.src & 15), ws = mis >> 2, bs = (mis & 3) * 8;
        const uint4 *asrc = (const uint4 *)(src - mis);
        uint4 *dst = (uint4 *)mm.dst;
        uint32_t y0 = 0, y1 = 0, y2 = 0, y3 = 0;
        uint64_t last = ~0ull;
        for (uint64_t bw = b0; bw <= e; bw += 32) {
            const uint64_t b = bw + lane;
            if (b > e) continue;
            // the block's 16 bytes (little-endian words), realigned from the aligned granules that hold them; a granule
            // is only read when it holds a byte of the range
            uint4 lo = asrc[b];
            uint32_t w0 = lo.x, w1 = lo.y, w2 = lo.z, w3 = lo.w;
            if (mis) {
                const uint4 hi = (16 * b + 16 - mis < mm.len) ? asrc[b + 1] : make_uint4(0, 0, 0, 0);
                const uint32_t v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
                uint32_t o[5];
#pragma unroll
                for (int k = 0; k < 5; k++) o[k] = ws == 0 ? v[k] : ws == 1 ? v[k + 1] : ws == 2 ? v[k + 2] : v[k + 3];
                w0 = __funnelshift_r(o[0], o[1], bs); w1 = __funnelshift_r(o[1], o[2], bs);
                w2 = __funnelshift_r(o[2], o[3], bs); w3 = __funnelshift_r(o[3], o[4], bs);
            }
            // keystream block E_K(inc32^(b+1)(J0))
            uint32_t s0 = mm.j0[0] ^ RK[0], s1 = mm.j0[1] ^ RK[1], s2 = mm.j0[2] ^ RK[2];
            uint32_t s3 = (mm.j0[3] + (uint32_t)b + 1u) ^ RK[3];
#pragma unroll
            for (int rd = 1; rd < 14; rd++) {
                const uint32_t a = GT(s0, 24) ^ rorr(GT(s1, 16), 8) ^ rorr(GT(s2, 8), 16) ^ rorr(GT(s3, 0), 24) ^ RK[4 * rd];
                const uint32_t bb = GT(s1, 24) ^ rorr(GT(s2, 16), 8) ^ rorr(GT(s3, 8), 16) ^ rorr(GT(s0, 0), 24) ^ RK[4 * rd + 1];
                const uint32_t c = GT(s2, 24) ^ rorr(GT(s3, 16), 8) ^ rorr(GT(s0, 8), 16) ^ rorr(GT(s1, 0), 24) ^ RK[4 * rd + 2];
                const uint32_t d = GT(s3, 24) ^ rorr(GT(s0, 16), 8) ^ rorr(GT(s1, 8), 16) ^ rorr(GT(s2, 0), 24) ^ RK[4 * rd + 3];
                s0 = a; s1 = bb; s2 = c; s3 = d;
            }
            // last round: the S-box is byte 2 of T0
#define LR(p, q, u, v) ((GT(p, 24) & 0x00FF0000u) << 8 | (GT(q, 16) & 0x00FF0000u) | (GT(u, 8) & 0x0000FF00u) | ((GT(v, 0) >> 8) & 0xFFu))
            const uint32_t k0 = LR(s0, s1, s2, s3) ^ RK[56], k1 = LR(s1, s2, s3, s0) ^ RK[57];
            const uint32_t k2 = LR(s2, s3, s0, s1) ^ RK[58], k3 = LR(s3, s0, s1, s2) ^ RK[59];
#undef LR
            uint32_t x0 = bswap32(w0), x1 = bswap32(w1), x2 = bswap32(w2), x3 = bswap32(w3);
            if (DECRYPT && 16 * b + 16 > mm.len) {   // the ciphertext is hashed: drop the bytes past the message (the next blob's)
                const int rv = (int)(mm.len - 16 * b);
                x0 &= keep_mask(rv, 0); x1 &= keep_mask(rv, 1); x2 &= keep_mask(rv, 2); x3 &= keep_mask(rv, 3);
            }
            uint32_t c0 = x0 ^ k0, c1 = x1 ^ k1, c2 = x2 ^ k2, c3 = x3 ^ k3;
            if (16 * b + 16 > mm.len) {   // partial last block: GHASH pads with zeros
                const int rv = (int)(mm.len - 16 * b);
                c0 &= keep_mask(rv, 0); c1 &= keep_mask(rv, 1); c2 &= keep_mask(rv, 2); c3 &= keep_mask(rv, 3);
            }
            dst[b] = make_uint4(bswap32(c0), bswap32(c1), bswap32(c2), bswap32(c3));
            // lane Horner with the step H^32, over the ciphertext: the output when encrypting, the input when decrypting
            uint32_t y[4] = {y0, y1, y2, y3};
            gf_mul_table(y, [&](uint32_t i) { return M32[i]; }, [&](uint32_t i) { return R8[i]; });
            if (DECRYPT) { y0 = y[0] ^ x0; y1 = y[1] ^ x1; y2 = y[2] ^ x2; y3 = y[3] ^ x3; }
            else { y0 = y[0] ^ c0; y1 = y[1] ^ c1; y2 = y[2] ^ c2; y3 = y[3] ^ c3; }
            last = b;
        }
        uint32_t q[4] = {0, 0, 0, 0};
        if (last != ~0ull) {   // relative to the segment's last block
            const uint32_t *hp = tab->hp[e - last];
            const uint32_t h[4] = {__ldg(hp), __ldg(hp + 1), __ldg(hp + 2), __ldg(hp + 3)};
            const uint32_t y[4] = {y0, y1, y2, y3};
            if (DECRYPT) gf_mul_reg(y, h, q);
            else gf_mul(y, h, q);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1)
#pragma unroll
            for (int k = 0; k < 4; k++) q[k] ^= __shfl_xor_sync(0xFFFFFFFFu, q[k], d);
        if (lane == 0) part[g] = make_uint4(q[0], q[1], q[2], q[3]);
    }
#undef GT
}

// one thread per message: chain its segments, add the length block, XOR E_K(J0); tag bytes to tags + 16 r
__global__ void k_gcm_tag(const GcmMsg *msg, const uint64_t *seg_first, uint32_t n, const GcmTables *tab,
                          const uint4 *part, uint8_t *tags) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const GcmMsg mm = msg[r];
    const uint64_t s0 = seg_first[r], ns = seg_first[r + 1] - s0, m = (mm.len + 15) >> 4;
    auto mt = [&](const uint32_t (*t)[4]) {
        return [t](uint32_t i) { return make_uint4(__ldg(&t[i][0]), __ldg(&t[i][1]), __ldg(&t[i][2]), __ldg(&t[i][3])); };
    };
    auto r8 = [tab](uint32_t i) { return __ldg(&tab->r8[i]); };
    uint32_t a[4] = {0, 0, 0, 0};
    for (uint64_t s = 0; s < ns; s++) {
        if (s) {
            const uint64_t k = s + 1 < ns ? GCM_SEG_BLOCKS : m - s * GCM_SEG_BLOCKS;   // blocks of segment s
            if (k == GCM_SEG_BLOCKS) gf_mul_table(a, mt(tab->mseg), r8);
            else {
                const uint32_t x[4] = {a[0], a[1], a[2], a[3]}, h[4] = {tab->hp[k][0], tab->hp[k][1], tab->hp[k][2], tab->hp[k][3]};
                gf_mul(x, h, a);
            }
        }
        const uint4 p = part[s0 + s];
        a[0] ^= p.x; a[1] ^= p.y; a[2] ^= p.z; a[3] ^= p.w;
    }
    // GHASH = (A * H ^ [0]_64 || [8 len]_64) * H
    gf_mul_table(a, mt(tab->m1), r8);
    const uint64_t bits = mm.len * 8;
    a[2] ^= (uint32_t)(bits >> 32); a[3] ^= (uint32_t)bits;
    gf_mul_table(a, mt(tab->m1), r8);
    for (int k = 0; k < 4; k++) {
        const uint32_t w = a[k] ^ mm.ej0[k];
        for (int i = 0; i < 4; i++) tags[16ull * r + 4 * k + i] = (uint8_t)(w >> (24 - 8 * i));
    }
}

uint64_t gcm_segments(uint64_t len) { return (((len + 15) >> 4) + GCM_SEG_BLOCKS - 1) / GCM_SEG_BLOCKS; }

cudaError_t launch_gcm(const GcmMsg *msg, const uint64_t *seg_first, uint32_t n, uint64_t total_segs, const void *tables,
                       void *part, uint8_t *tags, int sm_count, cudaStream_t st, bool decrypt) {
    if (n == 0) return cudaSuccess;
    if (total_segs) {
        auto kern = decrypt ? k_gcm_ctr_ghash<true> : k_gcm_ctr_ghash<false>;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GCM_SMEM);
        if (e != cudaSuccess) return e;
        const uint64_t want = (total_segs + GCM_THREADS / 32 - 1) / (GCM_THREADS / 32);
        const uint64_t cap = (uint64_t)sm_count * 4;
        kern<<<(unsigned)(want < cap ? want : cap), GCM_THREADS, GCM_SMEM, st>>>(
            msg, seg_first, n, total_segs, (const GcmTables *)tables, (uint4 *)part);
    }
    k_gcm_tag<<<(n + 127) / 128, 128, 0, st>>>(msg, seg_first, n, (const GcmTables *)tables, (const uint4 *)part, tags);
    return cudaGetLastError();
}

}  // namespace pbsgpu
