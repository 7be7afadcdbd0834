// pbs_plus_b200/csrc/scan.cu -- K1: buzhash boundary-candidate scan (sm_90a).
//
// Replaces the byte-at-a-time rolling-hash loop the reference runs inside
// transfer.ArchiveWriter.WriteEntryReader (reference internal/pxarmount/commit.go:720,
// :858; arithmetic = upstream PBS ChunkerImpl::scan).  The window is 64 bytes, so the
// hash at position i is position independent:
//     H(i) = XOR_{j=0..63} rotl32(T[b[i-j]], j mod 32)
// and every position can be tested in parallel.  K1 emits CANDIDATES (positions whose
// hash passes the break test); K2 (resolve.cu) applies the sequential min/max rule.
//
// Tuned kernel (k_scan_tuned), integer/byte work, no tensor cores:
//   * one warp owns a tile of 32 x 272 B; the tile (+64 B halo) is brought into shared
//     memory by ONE TMA bulk copy (device.cuh stage_bulk, SASS UBLKCP), double
//     buffered per warp, so HBM reads are fully coalesced and cost no issue slots;
//   * each lane walks its own 272 B span (64 B warm-up from the halo);
//   * de-rotated prefix form: A[p] = rotr(T[b[p]], (p+lane) mod 32), Q(p) = Q(p-1)^A[p],
//     G(p) = Q(p)^Q(p-64) = rotr(H(p), (p+lane) mod 32).  A[p] comes from a 64 KiB shared
//     table rot[b][slot] = rotr(T[b], slot mod 32), slot = (p mod 32) + lane: the bank
//     is (lane + p) mod 32 for every data byte -> conflict free by construction, and
//     the address is ONE PRMT (b<<8 | lane*4) plus an immediate;
//   * the 64-entry Q ring lives in registers; the break test is ONE instruction per
//     byte: LOP3.LUT.PAND  P &= ((~(Q^Qold) & rotr(M21,.)) != 0)   (M21 = mask & ~3);
//     only if P drops (p ~ 1e-4 per lane span) the lane re-walks its span exactly.
//   => 3 ALU-pipe instructions per byte (PRMT, XOR, LOP3.PAND) + 1 LDS.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

__device__ __forceinline__ uint32_t rotl32(uint32_t x, uint32_t r) { return __funnelshift_l(x, x, r); }
__device__ __forceinline__ uint32_t rotr32(uint32_t x, uint32_t r) { return __funnelshift_r(x, x, r); }

__device__ __forceinline__ void emit_candidate(const ScanArgs &a, uint32_t stream, uint64_t pos) {
    unsigned long long i = atomicAdd(a.cand_count, 1ull);
    if (i < a.cand_cap) a.cand[i] = ((uint64_t)stream << KEY_POS_BITS) | pos;
}

// ============================================================================
// Cross-check kernel: one thread per SIMPLE_SPAN bytes, plain rolling recurrence.
// Same results as the tuned kernel; used by tests and by variant==1.
// "tiles" here are SIMPLE_SPAN-byte spans (tile_first built with that size).
// ============================================================================
__global__ void __launch_bounds__(256) k_scan_simple(ScanArgs a) {
    __shared__ uint32_t T[256];
    T[threadIdx.x] = a.table[threadIdx.x];
    __syncthreads();
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.total_tiles) return;
    uint32_t s = owner_of(a.tile_first, a.n_streams, g);
    uint64_t j = g - a.tile_first[s];
    uint64_t len = a.len[s];
    const uint8_t *d = a.base + a.off[s];
    uint64_t start = j * SIMPLE_SPAN;
    uint64_t end = start + SIMPLE_SPAN < len ? start + SIMPLE_SPAN : len;
    uint64_t wstart = start >= 63 ? start - 63 : 0;
    uint32_t h = 0;
    for (uint64_t q = wstart; q < end; q++) {
        h = rotl32(h, 1) ^ T[d[q]];
        if (q >= wstart + 64) h ^= T[d[q - 64]];
        if (q >= start && q >= 63 && (h & a.mask) >= a.break_min) emit_candidate(a, s, q);
    }
}

cudaError_t launch_scan_simple(const ScanArgs &a, cudaStream_t st) {
    if (a.total_tiles == 0) return cudaSuccess;
    uint64_t blocks = (a.total_tiles + 255) / 256;
    k_scan_simple<<<(unsigned)blocks, 256, 0, st>>>(a);
    return cudaGetLastError();
}

// ============================================================================
// Tuned kernel
// ============================================================================
constexpr int HALO = 64;
constexpr int BUF_BYTES = HALO + WARP_TILE;            // 8768
constexpr int BUF_STRIDE = (BUF_BYTES + 127) & ~127;   // 8832
constexpr int WARPS_PER_CTA = 8;
constexpr int ROT_SLOTS = 64;
constexpr int ROT_BYTES = 256 * ROT_SLOTS * 4;         // 65536
constexpr int SMEM_BYTES = ROT_BYTES + WARPS_PER_CTA * 2 * BUF_STRIDE + WARPS_PER_CTA * 2 * 8;

size_t scan_tuned_smem_bytes() { return SMEM_BYTES; }

__global__ void k_build_rot_table(const uint32_t *table, uint32_t *rot) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;  // 256*64 entries
    if (i < 256 * ROT_SLOTS) rot[i] = rotr32(table[i >> 6], (i & 63) & 31);
}
cudaError_t launch_build_rot_table(const uint32_t *table, uint32_t *rot, cudaStream_t st) {
    k_build_rot_table<<<64, 256, 0, st>>>(table, rot);
    return cudaGetLastError();
}

// d = ~(a^b) & c ;  acc = (d != 0) & acc      -> one LOP3.LUT.PAND
__device__ __forceinline__ void test_acc(uint32_t a, uint32_t b, uint32_t c, uint32_t &acc) {
    asm("{ .reg .pred q, r; .reg .b32 d;\n setp.ne.u32 q, %0, 0;\n lop3.and.b32 d|r, %1, %2, %3, 0x82, q;\n"
        " selp.u32 %0, 1, 0, r; }"
        : "+r"(acc)
        : "r"(a), "r"(b), "r"(c));
}

// 64 bytes of one lane: 4 x LDS.128 of data, per byte PRMT -> LDS(rot) -> XOR (-> test).
// SWZ: the lane's 256 B piece lies in a SWIZZLE_128B tensor-map tile [half][lane][128 B]: vector V (0..15) of the piece
// is at row + (V >> 3) * 4096 + (((V & 7) ^ sw) << 4), sw = lane & 7 (`data` = row, `v0` = first vector of this block).
template <bool TEST, int NVEC, bool SWZ = false>
__device__ __forceinline__ void lane_block(const uint4 *data, const uint8_t *rotb, uint32_t laneoff, uint32_t (&Q)[64],
                                           const uint32_t (&M)[32], uint32_t &q, uint32_t &acc, uint32_t v0 = 0, uint32_t sw = 0) {
#pragma unroll
    for (int v = 0; v < NVEC; v++) {
        uint4 d;
        if (SWZ) {
            const uint32_t V = v0 + v;
            d = *(const uint4 *)((const uint8_t *)data + ((V >> 3) << 12) + (((V & 7) ^ sw) << 4));
        } else {
            d = data[v];
        }
        uint32_t w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int p = v * 16 + j;  // p mod 64 (blocks start at multiples of 64)
            uint32_t idx = __byte_perm(w[j >> 2], laneoff, 0x5504 | ((j & 3) << 4));  // b<<8 | lane*4
            uint32_t val = *(const uint32_t *)(rotb + idx + (p & 31) * 4);
            q ^= val;
            if (TEST) test_acc(q, Q[p], M[p & 31], acc);
            Q[p] = q;
        }
    }
}

struct TileInfo {
    uint32_t stream;
    uint32_t valid;      // bytes of the stream in this tile (1..WARP_TILE)
    uint64_t stream_pos; // stream offset of the tile's first byte
};

// Exact walk of one lane span (slow path: flagged lanes and partial tiles).
// buf points at the warp buffer (halo at [0,64), tile at [64, 64+valid)).
__device__ __noinline__ void lane_exact(const ScanArgs &a, const uint8_t *buf, const uint32_t *rot, uint32_t lane,
                                        const TileInfo &ti) {
    int v = (int)ti.valid - (int)lane * LANE_SPAN;
    if (v <= 0) return;
    if (v > LANE_SPAN) v = LANE_SPAN;
    const uint8_t *B = buf + lane * LANE_SPAN;  // halo start of this lane
    // T[b] = rotl(rot[b][lane], lane): per-lane slot keeps the lookups bank-conflict free
    uint32_t h = 0;
    for (int p = 0; p < 64; p++) h = rotl32(h, 1) ^ rotl32(rot[B[p] * ROT_SLOTS + lane], lane);
    for (int p = 64; p < 64 + v; p++) {
        h = rotl32(h, 1) ^ rotl32(rot[B[p] * ROT_SLOTS + lane], lane) ^ rotl32(rot[B[p - 64] * ROT_SLOTS + lane], lane);
        uint64_t pos = ti.stream_pos + (uint64_t)lane * LANE_SPAN + (uint32_t)(p - 64);
        if (pos >= 63 && (h & a.mask) >= a.break_min) emit_candidate(a, ti.stream, pos);
    }
}

// Dynamic shared memory of both TMA-fed kernels: 1024 B aligned for k_scan_lanes' SWIZZLE_128B boxes.
extern __shared__ __align__(1024) uint8_t smem[];

__global__ void __launch_bounds__(WARPS_PER_CTA * 32, 1) k_scan_tuned(ScanArgs a, const uint32_t *__restrict__ rot_g) {
    uint32_t *rot = (uint32_t *)smem;
    const uint8_t *rotb = smem;
    {   // 64 KiB table: coalesced 16 B loads, once per (persistent) CTA
        const uint4 *src = (const uint4 *)rot_g;
        uint4 *dst = (uint4 *)smem;
        for (int i = threadIdx.x; i < ROT_BYTES / 16; i += blockDim.x) dst[i] = src[i];
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *buf0 = smem + ROT_BYTES + warp * 2 * BUF_STRIDE;
    uint64_t *bars = (uint64_t *)(smem + ROT_BYTES + WARPS_PER_CTA * 2 * BUF_STRIDE) + warp * 2;
    const uint32_t bar_s[2] = {smem_u32(&bars[0]), smem_u32(&bars[1])};
    warp_bars_init(bar_s, lane);

    const uint64_t gw = (uint64_t)blockIdx.x * WARPS_PER_CTA + warp, nw = (uint64_t)gridDim.x * WARPS_PER_CTA;
    const uint64_t t0 = a.total_tiles * gw / nw, t1 = a.total_tiles * (gw + 1) / nw;
    if (t0 >= t1) return;

    // per-lane constants
    const uint32_t m21 = a.mask & ~3u;
    uint32_t M[32];
#pragma unroll
    for (int k = 0; k < 32; k++) M[k] = rotr32(m21, (k + lane) & 31);
    const uint32_t laneoff = lane * 4;

    // stream cursor (advances monotonically with t)
    uint32_t s = owner_of(a.tile_first, a.n_streams, t0);
    uint64_t s_first = a.tile_first[s], s_next = a.tile_first[s + 1];

    auto tile_info = [&](uint64_t t, uint32_t &sc, uint64_t &sf, uint64_t &sn) {
        while (t >= sn) { sc++; sf = sn; sn = a.tile_first[sc + 1]; }
        TileInfo ti;
        ti.stream = sc;
        uint64_t j = t - sf, len = a.len[sc];
        ti.stream_pos = j * WARP_TILE;
        uint64_t rem = len - ti.stream_pos;
        ti.valid = rem < (uint64_t)WARP_TILE ? (uint32_t)rem : (uint32_t)WARP_TILE;
        return ti;
    };
    // bring tile `ti` into buffer b (halo + data).  All lanes call this (converged).
    auto issue = [&](const TileInfo &ti, int b) {
        uint8_t *buf = buf0 + b * BUF_STRIDE;
        const uint8_t *src = a.base + a.off[ti.stream] + ti.stream_pos;
        uint32_t halo = ti.stream_pos ? HALO : 0;
        uint32_t bytes = halo + ti.valid;
        const uint8_t *src0 = src - halo;
        uint8_t *dst0 = buf + (HALO - halo);
        if (!halo && lane < 16) ((uint32_t *)buf)[lane] = 0;   // stream start: zero halo (never reported: pos < 63)
        if ((((uintptr_t)src0) & 15) == 0) {
            uint32_t bulk = bytes & ~15u;
            for (uint32_t i = bulk + lane; i < bytes; i += 32) dst0[i] = src0[i];   // < 16 tail bytes
            __syncwarp();
            if (lane == 0) stage_bulk(dst0, src0, bulk, bar_s[b]);
        } else {   // unaligned source: cooperative generic copy (slow path; TMA needs 16 B alignment)
            for (uint32_t i = lane; i < bytes; i += 32) dst0[i] = src0[i];
            __syncwarp();
            if (lane == 0) mbar_arrive_expect_tx(bar_s[b], 0);
        }
    };

    TileInfo cur = tile_info(t0, s, s_first, s_next);
    issue(cur, 0);
    for (uint64_t t = t0; t < t1; t++) {
        const int b = (int)((t - t0) & 1);
        const uint32_t parity = (uint32_t)(((t - t0) >> 1) & 1);
        TileInfo nxt = cur;
        if (t + 1 < t1) {
            nxt = tile_info(t + 1, s, s_first, s_next);
            issue(nxt, b ^ 1);
        }
        mbar_wait(bar_s[b], parity);
        const uint8_t *buf = buf0 + b * BUF_STRIDE;
        if (cur.valid == WARP_TILE) {
            uint32_t Q[64];
            uint32_t q = 0, acc = 1;
            const uint4 *data = (const uint4 *)(buf + lane * LANE_SPAN);
            lane_block<false, 4>(data, rotb, laneoff, Q, M, q, acc);   // halo: warm-up, no test
            // fully unrolled: in a rolled loop every byte costs an extra register move (the ring slot Q[p] must return to
            // its canonical register at the back-edge); unrolled, the renaming is free (65 -> ~10 IMAD.MOV per 64 B)
#pragma unroll
            for (int it = 1; it <= 4; it++) lane_block<true, 4>(data + it * 4, rotb, laneoff, Q, M, q, acc);
            lane_block<true, 1>(data + 20, rotb, laneoff, Q, M, q, acc);  // 272 = 4*64 + 16
            if (!acc) lane_exact(a, buf, rot, lane, cur);
        } else {
            lane_exact(a, buf, rot, lane, cur);
        }
        __syncwarp();
        cur = nxt;
    }
}

// ============================================================================
// Lane-contiguous variant (k_scan_lanes).  In k_scan_tuned a lane's 272 B span of the next tile is not
// adjacent to its span of this tile, so every tile pays a 64 B warm-up per lane (23.5 % extra work).
// Here a warp owns a SUPER-TILE of 32 x 2 KiB: lane L owns the contiguous bytes [L*2048, (L+1)*2048) and
// walks them in 8 steps of 256 B; each step brings 32 per-lane 256 B pieces by TMA (tools/tma_piece_probe:
// same HBM rate as one contiguous 8 KiB copy), and the lane's 64-entry Q ring simply carries over from
// step to step -- the warm-up is paid once per 2 KiB (3 %).  A stream's tail (< 64 KiB) and streams whose
// start is not 16 B aligned keep using plain 8704 B tiles inside the same kernel.
// tile_first[] then counts STEPS: 8 per super-tile (floor(len / 64 KiB) of them), then one per plain tile.
// ============================================================================
constexpr int LS_R = 2048;                    // bytes per lane per super-tile
constexpr int LS_PIECE = 256;
constexpr int LS_STEPS = LS_R / LS_PIECE;     // 8
constexpr int LS_SUPER = 32 * LS_R;           // 64 KiB
constexpr int LS_HALO_STRIDE = 64;            // per-lane halo rows behind the 8 KiB box (read 4 x per 8 steps: conflicts do not matter)
constexpr int LS_BUF = 10240;                 // step buffer: 8 KiB tensor-map box (1024 B aligned for SWIZZLE_128B) + 2 KiB halo;
                                              // a plain 8704 B tile (+64 B halo) fits too
constexpr int LS_BOX = 32 * LS_PIECE;         // 8192
constexpr int LS_SMEM = ROT_BYTES + WARPS_PER_CTA * 2 * LS_BUF + WARPS_PER_CTA * 2 * 8;
constexpr uint32_t LS_ALIGN = 128;            // a stream takes super-tiles only if it starts on a 128 B unit of the tensor map

uint64_t scan_lanes_super_bytes() { return LS_SUPER; }
uint32_t scan_lanes_align() { return LS_ALIGN; }
uint32_t scan_lanes_steps() { return LS_STEPS; }


// Exact walk of one lane's 256 B piece (slow path of k_scan_lanes).  The piece is in shared memory; the 64 bytes
// before it left shared memory a step ago, so they come back from global memory (L2) as four 16 B loads.
// `row` = the lane's 128 B row of half 0 in the swizzled tile; byte p of the piece is at
// row + (p >> 7) * 4096 + ((((p >> 4) & 7) ^ sw) << 4) + (p & 15).
__device__ __noinline__ void piece_exact(const ScanArgs &a, const uint8_t *row, const uint32_t *rot, uint32_t lane,
                                         uint32_t stream, const uint8_t *d, uint64_t start) {
    const uint32_t sw = lane & 7;
    auto piece_at = [&](int p) -> uint32_t { return row[((p >> 7) << 12) + ((((p >> 4) & 7) ^ sw) << 4) + (p & 15)]; };
    uint4 hv[4];
    if (start >= 64) {
        const uint4 *g = (const uint4 *)(d + start - 64);   // stream start and `start` are multiples of 16
#pragma unroll
        for (int i = 0; i < 4; i++) hv[i] = g[i];
    } else {
#pragma unroll
        for (int i = 0; i < 4; i++) hv[i] = make_uint4(0, 0, 0, 0);
    }
    const uint8_t *halo = (const uint8_t *)hv;
    uint32_t h = 0;
    for (int p = 0; p < 64; p++) h = rotl32(h, 1) ^ rotl32(rot[halo[p] * ROT_SLOTS + lane], lane);
    for (int p = 0; p < LS_PIECE; p++) {
        const uint32_t leave = p < 64 ? halo[p] : piece_at(p - 64);
        h = rotl32(h, 1) ^ rotl32(rot[piece_at(p) * ROT_SLOTS + lane], lane) ^ rotl32(rot[leave * ROT_SLOTS + lane], lane);
        const uint64_t pos = start + (uint32_t)p;
        if (pos >= 63 && (h & a.mask) >= a.break_min) emit_candidate(a, stream, pos);
    }
}

// 64 bytes whose four 16 B vectors the caller has loaded (lane-contiguous kernel: swizzled shared addresses)
template <bool TEST>
__device__ __forceinline__ void lane_block_v(const uint4 (&dv)[4], const uint8_t *rotb, uint32_t laneoff, uint32_t (&Q)[64],
                                             const uint32_t (&M)[32], uint32_t &q, uint32_t &acc) {
#pragma unroll
    for (int v = 0; v < 4; v++) {
        const uint32_t w[4] = {dv[v].x, dv[v].y, dv[v].z, dv[v].w};
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int p = v * 16 + j;
            uint32_t idx = __byte_perm(w[j >> 2], laneoff, 0x5504 | ((j & 3) << 4));  // b<<8 | lane*4
            uint32_t val = *(const uint32_t *)(rotb + idx + (p & 31) * 4);
            q ^= val;
            if (TEST) test_acc(q, Q[p], M[p & 31], acc);
            Q[p] = q;
        }
    }
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}

// Work unit of k_scan_lanes: a super-tile (8 steps) or a plain tile.
struct LsUnit {
    uint32_t stream;
    uint32_t kind;        // 0 = plain tile, 1 = super-tile
    uint32_t valid;       // plain tile: bytes of the stream in the tile
    uint64_t stream_pos;  // stream offset of the tile / super-tile
    uint64_t soff;        // a.off[stream]
};

__global__ void __launch_bounds__(WARPS_PER_CTA * 32, 1) k_scan_lanes(ScanArgs a, const uint32_t *__restrict__ rot_g,
                                                                       const __grid_constant__ CUtensorMap tmap) {
    uint32_t *rot = (uint32_t *)smem;
    const uint8_t *rotb = smem;
    {
        const uint4 *src = (const uint4 *)rot_g;
        uint4 *dst = (uint4 *)smem;
        for (int i = threadIdx.x; i < ROT_BYTES / 16; i += blockDim.x) dst[i] = src[i];
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *buf0 = smem + ROT_BYTES + warp * 2 * LS_BUF;          // ROT_BYTES = 64 KiB: every step buffer is 1024 B aligned
    uint64_t *bars = (uint64_t *)(smem + ROT_BYTES + WARPS_PER_CTA * 2 * LS_BUF) + warp * 2;
    const uint32_t bar_s[2] = {smem_u32(&bars[0]), smem_u32(&bars[1])};
    warp_bars_init(bar_s, lane);
    const uint64_t gw = (uint64_t)blockIdx.x * WARPS_PER_CTA + warp, nw = (uint64_t)gridDim.x * WARPS_PER_CTA;
    auto n_super_of = [&](uint32_t sc) -> uint64_t {
        return (a.off[sc] & (LS_ALIGN - 1)) == 0 ? a.len[sc] / LS_SUPER : 0;   // a.base itself is 128 B aligned (host checked)
    };
    // warps split the step list evenly, but a split inside a super-tile moves back to the super-tile's step 0
    auto round_unit = [&](uint64_t x) -> uint64_t {
        if (x >= a.total_tiles) return a.total_tiles;
        const uint32_t sc = owner_of(a.tile_first, a.n_streams, x);
        const uint64_t j = x - a.tile_first[sc];
        return j < n_super_of(sc) * LS_STEPS ? x - (j % LS_STEPS) : x;
    };
    const uint64_t u0 = round_unit(a.total_tiles * gw / nw), u1 = round_unit(a.total_tiles * (gw + 1) / nw);
    if (u0 >= u1) return;

    const uint32_t m21 = a.mask & ~3u;
    uint32_t M[32];
#pragma unroll
    for (int k = 0; k < 32; k++) M[k] = rotr32(m21, (k + lane) & 31);
    const uint32_t laneoff = lane * 4;
    // SWIZZLE_128B: 16 B chunk cc of the lane's 128 B row sits at (cc ^ (lane & 7)) << 4 -- eight per-lane constants
    uint32_t swz[8];
#pragma unroll
    for (int cc = 0; cc < 8; cc++) swz[cc] = ((uint32_t)cc ^ (lane & 7)) << 4;

    // unit cursor: tile_first[] counts STEPS (a super-tile is LS_STEPS of them, a plain tile one); all the bookkeeping
    // below runs once per UNIT (64 KiB), not once per step
    uint32_t s = owner_of(a.tile_first, a.n_streams, u0);
    uint64_t s_first = a.tile_first[s], s_next = a.tile_first[s + 1];
    uint64_t s_ns = n_super_of(s), s_off = a.off[s], s_len = a.len[s];
    uint64_t u = u0;
    auto next_unit = [&](LsUnit &un) -> bool {
        if (u >= u1) return false;
        while (u >= s_next) { s++; s_first = s_next; s_next = a.tile_first[s + 1]; s_ns = n_super_of(s); s_off = a.off[s]; s_len = a.len[s]; }
        const uint64_t j = u - s_first;
        un.stream = s; un.soff = s_off;
        if (j < s_ns * LS_STEPS) {
            un.kind = 1; un.valid = 0; un.stream_pos = (j / LS_STEPS) * LS_SUPER;
            u += LS_STEPS;
        } else {
            un.kind = 0;
            un.stream_pos = s_ns * LS_SUPER + (j - s_ns * LS_STEPS) * WARP_TILE;
            const uint64_t rem = s_len - un.stream_pos;
            un.valid = rem < (uint64_t)WARP_TILE ? (uint32_t)rem : (uint32_t)WARP_TILE;
            u += 1;
        }
        return true;
    };
    // step k of super-tile `un` into buffer b: ONE tensor-map copy brings the 256 B piece of every lane -- box {128 B, 1,
    // 32 lanes (stride 2 KiB), 2 halves}, SWIZZLE_128B -> shared [half][lane][128 B] (SASS UTMALDG); only step 0 adds the
    // per-lane 64 B halos.  The caller has made sure (syncwarp) that every lane is done with buffer b.
    auto issue_super = [&](const LsUnit &un, uint32_t k, int b) {
        uint8_t *buf = buf0 + b * LS_BUF;
        if (k == 0) {
            const uint64_t lane_start = un.stream_pos + (uint64_t)lane * LS_R;
            const bool first_of_stream = lane_start == 0;                  // only lane 0 of the stream's first super-tile
            uint8_t *halo = buf + LS_BOX + lane * LS_HALO_STRIDE;
            if (first_of_stream) {
                uint32_t *hz = (uint32_t *)halo;
#pragma unroll
                for (int i = 0; i < 16; i++) hz[i] = 0;                     // zero halo (positions < 63 are never reported)
            }
            const uint32_t any_first = __ballot_sync(0xffffffffu, first_of_stream);
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                mbar_arrive_expect_tx(bar_s[b], LS_BOX + (32 - __popc(any_first)) * 64);
                tma_tensor4d_g2s(smem_u32(buf), &tmap, 0, (int)((un.soff + un.stream_pos) >> 7), 0, 0, bar_s[b]);
            }
            __syncwarp();
            if (!first_of_stream) tma_bulk_g2s(smem_u32(halo), a.base + un.soff + lane_start - 64, 64, bar_s[b]);
        } else if (lane == 0) {
            fence_proxy_async();
            mbar_arrive_expect_tx(bar_s[b], LS_BOX);
            const int c1 = (int)((un.soff + un.stream_pos + (uint64_t)k * LS_PIECE) >> 7);   // 128 B unit of lane 0's piece
            tma_tensor4d_g2s(smem_u32(buf), &tmap, 0, c1, 0, 0, bar_s[b]);
        }
    };
    // a plain tile: k_scan_tuned's `issue` written out again -- one function shared by both kernels raises this kernel
    // from 208 to 212-214 registers
    auto issue_plain = [&](const LsUnit &un, int b) {
        uint8_t *buf = buf0 + b * LS_BUF;
        const uint8_t *src = a.base + un.soff + un.stream_pos;
        uint32_t halo = un.stream_pos ? HALO : 0;
        uint32_t bytes = halo + un.valid;
        const uint8_t *src0 = src - halo;
        uint8_t *dst0 = buf + (HALO - halo);
        if (!halo && lane < 16) ((uint32_t *)buf)[lane] = 0;
        if ((((uintptr_t)src0) & 15) == 0) {
            uint32_t bulk = bytes & ~15u;
            for (uint32_t i = bulk + lane; i < bytes; i += 32) dst0[i] = src0[i];
            __syncwarp();
            if (lane == 0) stage_bulk(dst0, src0, bulk, bar_s[b]);
        } else {
            for (uint32_t i = lane; i < bytes; i += 32) dst0[i] = src0[i];
            __syncwarp();
            if (lane == 0) mbar_arrive_expect_tx(bar_s[b], 0);
        }
    };
    auto issue_first = [&](const LsUnit &un, int b) { if (un.kind == 1) issue_super(un, 0, b); else issue_plain(un, b); };

    uint32_t Q[64];
    uint32_t q = 0;
    LsUnit cur, nxt;
    bool have = next_unit(cur);
    if (have) issue_first(cur, 0);
    uint32_t n = 0;   // steps processed by this warp: buffer = n & 1, mbarrier parity = (n >> 1) & 1
    while (have) {
        const bool have_next = next_unit(nxt);
        if (cur.kind == 1) {
#pragma unroll 1
            for (uint32_t k = 0; k < LS_STEPS; k++, n++) {
                const int b = (int)(n & 1);
                if (k + 1 < LS_STEPS) issue_super(cur, k + 1, b ^ 1);
                else if (have_next) issue_first(nxt, b ^ 1);
                mbar_wait(bar_s[b], (n >> 1) & 1);
                const uint8_t *buf = buf0 + b * LS_BUF;
                uint32_t acc = 1;
                if (k == 0) {
                    q = 0;
                    lane_block<false, 4>((const uint4 *)(buf + LS_BOX + lane * LS_HALO_STRIDE), rotb, laneoff, Q, M, q, acc);
                }
                const uint32_t row = smem_u32(buf) + lane * 128;          // the lane's row of half 0 in the swizzled tile
                uint32_t ad[8];
#pragma unroll
                for (int cc = 0; cc < 8; cc++) ad[cc] = row + swz[cc];
#pragma unroll
                for (int it = 0; it < 4; it++) {                            // 4 x 64 B, all addresses compile-time + ad[]
                    uint4 dv[4];
#pragma unroll
                    for (int v = 0; v < 4; v++) {
                        const int V = it * 4 + v;
                        dv[v] = lds128(ad[V & 7] + ((V >> 3) << 12));
                    }
                    lane_block_v<true>(dv, rotb, laneoff, Q, M, q, acc);
                }
                if (!acc)
                    piece_exact(a, buf + lane * 128, rot, lane, cur.stream, a.base + cur.soff,
                                cur.stream_pos + (uint64_t)lane * LS_R + (uint64_t)k * LS_PIECE);
                __syncwarp();
            }
        } else {
            const int b = (int)(n & 1);
            if (have_next) issue_first(nxt, b ^ 1);
            mbar_wait(bar_s[b], (n >> 1) & 1);
            const uint8_t *buf = buf0 + b * LS_BUF;
            uint32_t acc = 1;
            TileInfo ti;
            ti.stream = cur.stream; ti.valid = cur.valid; ti.stream_pos = cur.stream_pos;
            if (cur.valid == WARP_TILE) {
                const uint4 *data = (const uint4 *)(buf + lane * LANE_SPAN);
                q = 0;
                lane_block<false, 4>(data, rotb, laneoff, Q, M, q, acc);
#pragma unroll 1
                for (int it = 1; it <= 4; it++) lane_block<true, 4>(data + it * 4, rotb, laneoff, Q, M, q, acc);
                lane_block<true, 1>(data + 20, rotb, laneoff, Q, M, q, acc);
                if (!acc) lane_exact(a, buf, rot, lane, ti);
            } else {
                lane_exact(a, buf, rot, lane, ti);
            }
            __syncwarp();
            n++;
        }
        cur = nxt;
        have = have_next;
    }
}

typedef CUresult (*tmap_encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                   const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// `extent` = bytes of the batch buffer behind a.base that streams may touch (max off + len).  a.base must be 128 B aligned
// (the caller routes other bases to k_scan_tuned).
cudaError_t launch_scan_lanes(const ScanArgs &a, const uint32_t *rot_table, int sm_count, uint64_t extent, cudaStream_t st) {
    if (a.total_tiles == 0) return cudaSuccess;
    static tmap_encode_fn encode = nullptr;
    if (!encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn ||
            qr != cudaDriverEntryPointSuccess) { (void)cudaGetLastError(); return cudaErrorNotSupported; }
        encode = (tmap_encode_fn)fn;
    }
    // u8 tensor over the batch: dim0 = 128 contiguous bytes, dim1 = 128 B unit index, dim2 = lane (stride 2 KiB),
    // dim3 = half (stride 128 B); overlapping strides on purpose
    CUtensorMap tmap;
    const cuuint64_t units = extent / 128 ? extent / 128 : 1;
    const cuuint64_t dims[4] = {128, units, 32, 2};
    const cuuint64_t strides[3] = {128, LS_R, 128};
    const cuuint32_t box[4] = {128, 1, 32, 2}, estr[4] = {1, 1, 1, 1};
    if (encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, (void *)a.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return cudaErrorInvalidValue;
    cudaError_t e = cudaFuncSetAttribute(k_scan_lanes, cudaFuncAttributeMaxDynamicSharedMemorySize, LS_SMEM);
    if (e != cudaSuccess) return e;
    uint64_t want = (a.total_tiles + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    unsigned grid = (unsigned)(want < (uint64_t)sm_count ? want : (uint64_t)sm_count);
    k_scan_lanes<<<grid, WARPS_PER_CTA * 32, LS_SMEM, st>>>(a, rot_table, tmap);
    return cudaGetLastError();
}

cudaError_t launch_scan_tuned(const ScanArgs &a, const uint32_t *rot_table, int sm_count, cudaStream_t st) {
    if (a.total_tiles == 0) return cudaSuccess;
    // per launch (cheap): the attribute is per device and a process may drive several devices
    cudaError_t e = cudaFuncSetAttribute(k_scan_tuned, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return e;
    uint64_t want = (a.total_tiles + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    unsigned grid = (unsigned)(want < (uint64_t)sm_count ? want : (uint64_t)sm_count);
    k_scan_tuned<<<grid, WARPS_PER_CTA * 32, SMEM_BYTES, st>>>(a, rot_table);
    return cudaGetLastError();
}

}  // namespace pbsgpu
