// pbs_plus_b200/csrc/crc32.cu -- K6: batched CRC-32 (IEEE 802.3, zlib's crc32) of byte ranges.
//
// "Next" row f3 of SURVEY.md section 8: every NEW chunk is uploaded as a PBS DataBlob =
// { magic[8], crc32 LE of the payload, payload } (upstream pbs-datastore file_formats.rs /
// data_blob.rs; endpoints named at reference internal/server/backup/log_cleanup.go:19-31).  The
// payload bytes are already on the host; what the GPU adds is the checksum, another full pass over
// the new data.  zstd compression of blobs is out of scope (no compressor here).
//
// CRC is linear over GF(2), so a range is cut into regions hashed independently (k_crc32_tiled)
// and the partial CRCs are merged with zlib's crc32_combine algebra:
// crc(A||B) = crc(A) * x^(8|B|) mod P  xor  crc(B).
#include <cuda_runtime.h>
#include <stdint.h>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

constexpr uint32_t CRC_POLY = 0xedb88320u;   // reflected IEEE polynomial

// a(x) * b(x) mod P in the reflected representation (zlib multmodp)
__host__ __device__ inline uint32_t crc_multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}
// x^(n * 2^k) mod P, with x2n[i] = x^(2^i) mod P
__host__ __device__ inline uint32_t crc_x2nmodp(const uint32_t *x2n, uint64_t n, unsigned k) {
    uint32_t p = 1u << 31;
    while (n) {
        if (n & 1) p = crc_multmodp(x2n[k & 31], p);
        n >>= 1;
        k++;
    }
    return p;
}

struct CrcTables {
    uint32_t t[4][256];   // slicing-by-4
    uint32_t x2n[32];     // x^(2^i) mod P
};

void crc_make_tables(CrcTables *h) {
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
        h->t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; i++)
        for (int s = 1; s < 4; s++) h->t[s][i] = (h->t[s - 1][i] >> 8) ^ h->t[0][h->t[s - 1][i] & 0xff];
    uint32_t p = 1u << 30;   // x^1
    h->x2n[0] = p;
    for (int i = 1; i < 32; i++) h->x2n[i] = p = crc_multmodp(p, p);
}

// ============================================================================
// k_crc32_tiled: a warp owns REGIONS of 128 contiguous tiles of 32 x 144 B that arrive by TMA bulk copies
// (double buffered, as in the scan kernel), each lane walks its 144 B span of every tile (LDS.128, conflict
// free: lane stride = 9 quads) and carries its CRC state across tiles: the 4464 bytes of the other lanes
// between two of its spans are skipped with ONE table step (the "advance by n zero bytes" map is linear:
// 4 lookups).  At the end of a region every lane advances its
// state to the region end (one GF(2) multiplication) and the 32 states are XORed -- CRC is linear, the
// all-ones initial state rides on lane 0.  A range's unaligned head (< 16 B, TMA needs 16 B alignment) is
// hashed byte-wise by lane 0 in front of its first span.
// ============================================================================
constexpr int CT_SPAN = 144;                       // 9 x 16 B
constexpr int CT_TILE = 32 * CT_SPAN;              // 4608 B
constexpr int CT_REGION_TILES = 128;               // 576 KiB per region
constexpr int CT_WARPS = 8;
constexpr int CT_SMEM = 4 * 256 * 32 * 4 /*TR*/ + 4 * 256 * 4 /*ZT*/ + 4 * 256 * 4 /*T plain*/ + 32 * 4 +
                        CT_WARPS * 2 * CT_TILE + CT_WARPS * 2 * 8;

struct CrcTiledTables {
    CrcTables base;
    uint32_t zt[4][256];   // state advance by (CT_TILE - CT_SPAN) zero bytes, per state byte
};

// region_first[r] = first region index of range r (prefix over ceil(tiles/CT_REGION_TILES), >= 1 per
// non-empty range); part_crc[region] = standard CRC-32 of that region's bytes.
__global__ void __launch_bounds__(CT_WARPS * 32, 1) k_crc32_tiled(const uint8_t *base, const uint64_t *off,
                                                                  const uint64_t *len, const uint64_t *region_first,
                                                                  uint32_t n, uint64_t total_regions,
                                                                  const CrcTiledTables *tab, uint32_t *part_crc) {
    extern __shared__ __align__(128) uint8_t ct_smem[];
    uint32_t *TR = (uint32_t *)ct_smem;                       // [4][256][32]
    uint32_t *ZT = TR + 4 * 256 * 32;                         // [4][256]
    uint32_t *TP = ZT + 4 * 256;                              // [4][256] plain slicing tables (byte-wise paths)
    uint32_t *X2N = TP + 4 * 256;
    uint8_t *bufs = (uint8_t *)(X2N + 32);
    uint64_t *bars = (uint64_t *)(bufs + CT_WARPS * 2 * CT_TILE);
    for (int i = threadIdx.x; i < 4 * 256 * 32; i += blockDim.x) TR[i] = tab->base.t[i >> 13][(i >> 5) & 255];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) { ZT[i] = tab->zt[i >> 8][i & 255]; TP[i] = tab->base.t[i >> 8][i & 255]; }
    if (threadIdx.x < 32) X2N[threadIdx.x] = tab->base.x2n[threadIdx.x];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, lane4 = lane << 2;
    uint8_t *buf0 = bufs + warp * 2 * CT_TILE;
    const uint32_t bar_s[2] = {smem_u32(&bars[warp * 2]), smem_u32(&bars[warp * 2 + 1])};
    warp_bars_init(bar_s, lane);
    const uint8_t *TB = (const uint8_t *)TR;
    auto lut = [&](uint32_t k, uint32_t byte_shl7) -> uint32_t {
        return *(const uint32_t *)(TB + k * 32768u + ((byte_shl7 & 0x7f80u) | lane4));
    };
#define CT_BYTE(b) do { c = TP[(c ^ (b)) & 0xff] ^ (c >> 8); } while (0)
#define CT_WORD(w) do { c ^= (w); c = lut(3, c << 7) ^ lut(2, c >> 1) ^ lut(1, c >> 9) ^ lut(0, c >> 17); } while (0)
    uint32_t uses[2] = {0, 0};                                // per-buffer use counters (mbarrier phase parity)
    const uint64_t warps_total = (uint64_t)gridDim.x * CT_WARPS;
    for (uint64_t g = (uint64_t)blockIdx.x * CT_WARPS + warp; g < total_regions; g += warps_total) {
        const uint32_t r = owner_of(region_first, n, g);
        const uint64_t reg = g - region_first[r], rlen = len[r];
        const uint8_t *rstart = base + off[r];
        const uint32_t head = (uint32_t)((16 - ((uintptr_t)rstart & 15)) & 15);     // bytes before the aligned body
        const uint64_t head_eff = head < rlen ? head : rlen;
        const uint64_t body = rlen - head_eff;                                       // aligned part, tiled
        const uint64_t r_begin = reg * (uint64_t)CT_REGION_TILES * CT_TILE;          // body offset of this region
        const uint64_t r_bytes = body - r_begin < (uint64_t)CT_REGION_TILES * CT_TILE ? body - r_begin
                                                                                      : (uint64_t)CT_REGION_TILES * CT_TILE;
        const uint8_t *rbody = rstart + head_eff + r_begin;
        const uint32_t ntiles = (uint32_t)((r_bytes + CT_TILE - 1) / CT_TILE);
        // lane state and the body offset (within the region) up to which it has consumed bytes
        uint32_t c = 0;
        uint64_t consumed_end = (uint64_t)lane * CT_SPAN;      // where this lane's next span starts
        if (lane == 0) {
            c = 0xffffffffu;
            if (reg == 0) for (uint32_t i = 0; i < head_eff; i++) CT_BYTE(rstart[i]);   // unaligned head
        }
        bool started = false;                                   // lane has consumed a span of this region
        auto issue = [&](uint32_t t, int b) {
            const uint64_t tb = (uint64_t)t * CT_TILE;
            const uint32_t valid = r_bytes - tb < (uint64_t)CT_TILE ? (uint32_t)(r_bytes - tb) : (uint32_t)CT_TILE;
            const uint8_t *src = rbody + tb;
            uint8_t *dst = buf0 + b * CT_TILE;
            const uint32_t bulk = valid & ~15u;
            for (uint32_t i = bulk + lane; i < valid; i += 32) dst[i] = src[i];
            __syncwarp();
            if (lane == 0) stage_bulk(dst, src, bulk, bar_s[b]);
        };
        if (ntiles) issue(0, 0);
        for (uint32_t t = 0; t < ntiles; t++) {
            const int b = (int)(t & 1);
            if (t + 1 < ntiles) issue(t + 1, b ^ 1);
            mbar_wait(bar_s[b], uses[b] & 1);
            uses[b]++;
            const uint64_t tb = (uint64_t)t * CT_TILE;
            const uint32_t valid = r_bytes - tb < (uint64_t)CT_TILE ? (uint32_t)(r_bytes - tb) : (uint32_t)CT_TILE;
            const int v = (int)valid - (int)lane * CT_SPAN;     // bytes of this lane's span in the tile
            if (v > 0) {
                if (started)                                    // skip the other lanes' 4464 bytes since my last span
                    c = ZT[c & 0xff] ^ ZT[256 + ((c >> 8) & 0xff)] ^ ZT[512 + ((c >> 16) & 0xff)] ^ ZT[768 + (c >> 24)];
                started = true;
                const uint8_t *sp = buf0 + b * CT_TILE + lane * CT_SPAN;
                if (v >= CT_SPAN) {
                    const uint4 *q = (const uint4 *)sp;
#pragma unroll
                    for (int k = 0; k < CT_SPAN / 16; k++) {
                        uint4 d = q[k];
                        CT_WORD(d.x); CT_WORD(d.y); CT_WORD(d.z); CT_WORD(d.w);
                    }
                    consumed_end = tb + (uint64_t)lane * CT_SPAN + CT_SPAN;
                } else {
                    int i = 0;
                    for (; i + 4 <= v; i += 4) CT_WORD(*(const uint32_t *)(sp + i));
                    for (; i < v; i++) CT_BYTE(sp[i]);
                    consumed_end = tb + (uint64_t)lane * CT_SPAN + (uint32_t)v;
                }
            }
            __syncwarp();
        }
        // advance every lane's state to the region end and fold the 32 states (linearity)
        const uint64_t gap = started ? r_bytes - consumed_end : 0;   // lanes that never started hold 0 (or the
        if (gap && c) c = crc_multmodp(crc_x2nmodp(X2N, gap, 3), c);  // head-only state of lane 0): nothing to skip
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, d);
        if (lane == 0) part_crc[g] = ~c;
    }
#undef CT_WORD
#undef CT_BYTE
}

// one thread per range: merge its regions (variable first-region length because of the unaligned head)
__global__ void k_crc32_merge_regions(const uint8_t *base, const uint64_t *off, const uint64_t *len,
                                      const uint64_t *region_first, uint32_t n, const CrcTiledTables *tab,
                                      const uint32_t *part_crc, uint32_t *out) {
    uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint64_t g0 = region_first[r], g1 = region_first[r + 1], rlen = len[r];
    const uint32_t head = (uint32_t)((16 - ((uintptr_t)(base + off[r]) & 15)) & 15);
    const uint64_t head_eff = head < rlen ? head : rlen, body = rlen - head_eff;
    const uint64_t RB = (uint64_t)CT_REGION_TILES * CT_TILE;
    uint32_t acc = 0;
    for (uint64_t g = g0; g < g1; g++) {
        uint64_t k = g - g0;
        uint64_t bytes = body - k * RB < RB ? body - k * RB : RB;
        if (k == 0) bytes += head_eff;                         // region 0 also covers the head
        uint32_t f = crc_x2nmodp(tab->base.x2n, bytes, 3);
        acc = crc_multmodp(f, acc) ^ part_crc[g];
    }
    out[r] = acc;
}

cudaError_t launch_crc32_tiled(const uint8_t *base, const uint64_t *off, const uint64_t *len,
                               const uint64_t *region_first, uint32_t n, uint64_t total_regions, const void *tables,
                               uint32_t *part_crc, uint32_t *out, int sm_count, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    if (total_regions) {
        cudaError_t e = cudaFuncSetAttribute(k_crc32_tiled, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
        if (e != cudaSuccess) return e;
        uint64_t want = (total_regions + CT_WARPS - 1) / CT_WARPS;
        unsigned grid = (unsigned)(want < (uint64_t)sm_count ? want : (uint64_t)sm_count);
        k_crc32_tiled<<<grid, CT_WARPS * 32, CT_SMEM, st>>>(base, off, len, region_first, n, total_regions,
                                                           (const CrcTiledTables *)tables, part_crc);
    }
    k_crc32_merge_regions<<<(n + 127) / 128, 128, 0, st>>>(base, off, len, region_first, n,
                                                           (const CrcTiledTables *)tables, part_crc, out);
    return cudaGetLastError();
}
uint64_t crc_region_bytes() { return (uint64_t)CT_REGION_TILES * CT_TILE; }

size_t crc_tables_bytes() { return sizeof(CrcTiledTables); }
void crc_fill_tables_host(void *dst) {
    CrcTiledTables *t = (CrcTiledTables *)dst;
    crc_make_tables(&t->base);
    const uint32_t f = crc_x2nmodp(t->base.x2n, CT_TILE - CT_SPAN, 3);   // x^(8 * 4464)
    for (int k = 0; k < 4; k++)
        for (uint32_t b = 0; b < 256; b++) t->zt[k][b] = crc_multmodp(f, b << (8 * k));
}

}  // namespace pbsgpu
