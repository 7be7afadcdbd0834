// f3: the LZ77 match stage and Predefined_Mode sequences of compressed DataBlobs (K9, sm_90a).
//
// Every 128 KiB block of a chunk that is not one repeated byte (K8a decides that) becomes a zstd Compressed_Block
// (RFC 8878 3.1.1.3): a greedy LZ77 parse inside the block, Raw_Literals and a sequences section whose three FSE tables
// are the predefined ones.  The host (capi_aux.cu, zstd_frames) keeps that block when it is smaller than the raw one.
// The output is a pure function of the block's bytes; tests/zstd_lz_ref.py (zstd_frame_lz) states it.
//
//   cand(i)   for i <= S-4: the largest j in an EARLIER tile of LZ_TILE positions with h(j) == h(i), where
//             h(i) = (u32 LE at i * 0x9E3779B1) >> (32 - LZ_HBITS).  A tile looks up all of its positions before it
//             inserts any (atomicMax), so cand does not depend on the order of the threads.
//   match at i: cand(i) exists and the first LZ_MINMATCH bytes at cand(i) and i are equal (inside the block); its
//             length is the longest common extension inside the block (it may overlap i).
//   parse     from i = 0: at a match emit (literal run, length, i - cand(i)) and jump past it, else i + 1.
//
//   K9a k_lz_parse  : one CTA of 256 threads per block.  Per tile: every thread looks up one position into the shared
//                     cand[] tile, then inserts it; warp 0 then parses the tile -- a ballot finds the next match among
//                     32 positions, the literals before it are copied one byte per lane into the block's slot, and the
//                     match is extended 32 bytes per step.  Shared memory is the 32 KiB hash table + 1 KiB of cand, so
//                     six blocks are parsed at once per SM.  Sequences go to a per-pass scratch as packed u64.
//   K9b k_lz_encode : one THREAD per block (the backward FSE bitstream is serial by construction): literals header in
//                     front of the literals, the sequences header, the modes byte and the bitstream, behind them in the
//                     slot.  The tables sit in shared memory; the 32 blocks of a warp run in step.
#include "internal.cuh"

#include <cstring>

namespace pbsgpu {

constexpr int LZ_THREADS = 256;
static_assert(LZ_TILE == LZ_THREADS, "one position per thread per tile");

__device__ __forceinline__ uint32_t lz_key(const uint8_t *p) {
    return (uint32_t)__ldg(p) | (uint32_t)__ldg(p + 1) << 8 | (uint32_t)__ldg(p + 2) << 16 | (uint32_t)__ldg(p + 3) << 24;
}

__global__ void __launch_bounds__(LZ_THREADS) k_lz_parse(const uint8_t *base, const uint64_t *src, const uint32_t *size,
                                                         uint64_t first, uint8_t *slots, uint64_t *seqs, uint32_t *nseq,
                                                         uint32_t *nlit) {
    __shared__ int table[1 << LZ_HBITS];
    __shared__ int cand[LZ_TILE];
    const uint64_t g = first + blockIdx.x;
    const uint8_t *p = base + src[g];
    const uint32_t S = size[g];
    uint8_t *lit = slots + g * LZ_SLOT + 3;
    uint64_t *sq = seqs + (uint64_t)blockIdx.x * LZ_MAX_SEQ;
    const uint32_t lane = threadIdx.x & 31;
    const bool parser = threadIdx.x < 32;
    for (int k = threadIdx.x; k < (1 << LZ_HBITS); k += LZ_THREADS) table[k] = -1;
    __syncthreads();
    const uint32_t nk = S >= 4 ? S - 3 : 0;
    uint32_t pos = 0, run = 0, nl = 0, ns = 0;   // parser state (warp 0, the same in every lane)
    for (uint32_t t0 = 0; t0 < nk; t0 += LZ_TILE) {
        const uint32_t tend = min(t0 + LZ_TILE, nk);
        const uint32_t i = t0 + threadIdx.x;
        uint32_t h = 0;
        if (i < tend) {
            const uint32_t key = lz_key(p + i);
            h = (key * 0x9E3779B1u) >> (32 - LZ_HBITS);
            const int c = table[h];
            bool m = c >= 0 && lz_key(p + c) == key;
#pragma unroll
            for (int e = 4; e < LZ_MINMATCH; e++) m = m && i + e < S && __ldg(p + c + e) == __ldg(p + i + e);
            cand[threadIdx.x] = m ? c : -1;
        }
        __syncthreads();
        if (i < tend) atomicMax(&table[h], (int)i);
        if (parser) {
            while (pos < tend) {
                const uint32_t q = pos + lane;
                const uint32_t hits = __ballot_sync(~0u, q < tend && cand[q - t0] >= 0);
                const uint32_t m = hits ? pos + __ffs(hits) - 1 : min(pos + 32, tend);
                if (q < m) lit[nl + lane] = __ldg(p + q);
                nl += m - pos;
                pos = m;
                if (!hits) continue;
                const uint32_t c = (uint32_t)cand[m - t0];
                uint32_t L = LZ_MINMATCH;
                for (;;) {
                    const uint32_t a = m + L + lane;
                    const uint32_t diff = __ballot_sync(~0u, a >= S || __ldg(p + c + L + lane) != __ldg(p + a));
                    if (diff) { L += __ffs(diff) - 1; break; }
                    L += 32;
                }
                if (lane == 0) sq[ns] = (uint64_t)(m - run) | (uint64_t)L << 20 | (uint64_t)(m - c) << 40;
                ns++;
                pos = run = m + L;
            }
        }
        __syncthreads();   // cand[] is rewritten by the next tile
    }
    if (parser) {
        for (; pos < S; pos += 32) {
            if (pos + lane < S) lit[nl + lane] = __ldg(p + pos + lane);
            nl += min(32u, S - pos);
        }
        if (lane == 0) { nseq[g] = ns; nlit[g] = nl; }
    }
}

cudaError_t launch_lz_parse(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint64_t first, uint32_t nb,
                            uint8_t *slots, uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    k_lz_parse<<<nb, LZ_THREADS, 0, st>>>(base, src, size, first, slots, seqs, nseq, nlit);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(128) k_lz_encode(const LzTables *tab, uint64_t first, uint32_t nb, uint8_t *slots,
                                                   const uint64_t *seqs, const uint32_t *nseq, const uint32_t *nlit,
                                                   uint32_t *info) {
    __shared__ LzTables T;
    for (uint32_t k = threadIdx.x; k < sizeof(LzTables) / 16; k += blockDim.x) ((uint4 *)&T)[k] = ((const uint4 *)tab)[k];
    __syncthreads();
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const uint64_t g = first + b;
    const uint32_t n = nseq[g], nl = nlit[g];
    const uint32_t hl = nl <= 31 ? 1 : nl <= 4095 ? 2 : 3;   // Raw_Literals_Block header, Size_Format 00 / 01 / 11
    LzBits w{slots + g * LZ_SLOT, 3 - hl};
    if (hl == 1) w.byte(nl << 3);
    else if (hl == 2) { w.byte((nl << 4) | 0x4); w.byte(nl >> 4); }
    else { w.byte((nl << 4) | 0xC); w.byte(nl >> 4); w.byte(nl >> 12); }
    w.q = 3 + nl;
    if (n == 0) w.byte(0);
    else {
        if (n < 128) w.byte(n);
        else if (n < 0x7F00) { w.byte((n >> 8) + 0x80); w.byte(n & 0xFF); }
        else { w.byte(0xFF); w.byte((n - 0x7F00) & 0xFF); w.byte((n - 0x7F00) >> 8); }
        w.byte(0);   // Symbol_Compression_Modes: all Predefined_Mode
        const uint64_t *sq = seqs + (uint64_t)b * LZ_MAX_SEQ;
        uint32_t sLL = 0, sML = 0, sOF = 0;
        for (uint32_t k = n; k-- > 0;) {   // last sequence first
            const uint64_t s = sq[k];
            const uint32_t ll = (uint32_t)(s & 0xFFFFF), ml = (uint32_t)((s >> 20) & 0xFFFFF), ov = (uint32_t)(s >> 40) + 3;
            const uint32_t lc = ll < 64 ? T.ll_code[ll] : 31 - __clz(ll) + 19;
            const uint32_t mc = ml - 3 < 128 ? T.ml_code[ml - 3] : 31 - __clz(ml - 3) + 36;
            const uint32_t oc = 31 - __clz(ov);
            if (k + 1 == n) {
                sLL = T.ll_enc[lc][0] & 63; sML = T.ml_enc[mc][0] & 63; sOF = T.of_enc[oc][0] & 63;
            } else {   // the states from which the decoder reads this sequence's codes and then goes to the next one's
                uint32_t e = T.of_enc[oc][sOF]; w.add(e >> 9, (e >> 6) & 7); sOF = e & 63;
                e = T.ml_enc[mc][sML]; w.add(e >> 9, (e >> 6) & 7); sML = e & 63;
                e = T.ll_enc[lc][sLL]; w.add(e >> 9, (e >> 6) & 7); sLL = e & 63;
            }
            w.add(ll - T.ll_base[lc], T.ll_bits[lc]);
            w.add(ml - T.ml_base[mc], T.ml_bits[mc]);
            w.add(ov - (1u << oc), oc);
        }
        w.add(sML, 6); w.add(sOF, 5); w.add(sLL, 6); w.add(1, 1);
        if (w.n) w.byte((uint32_t)w.acc);
    }
    info[g] = (w.q - (3 - hl)) | (3 - hl) << 30;
}

cudaError_t launch_lz_encode(const LzTables *tab, uint64_t first, uint32_t nb, uint8_t *slots, const uint64_t *seqs,
                             const uint32_t *nseq, const uint32_t *nlit, uint32_t *info, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    k_lz_encode<<<(nb + 127) / 128, 128, 0, st>>>(tab, first, nb, slots, seqs, nseq, nlit, info);
    return cudaGetLastError();
}

// ---- host: the predefined tables (RFC 8878 3.1.1.3.2.2 distributions, 4.1.1 table construction) ----------------------
static const int LL_NORM[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1,
                                -1, -1, -1, -1};
static const int ML_NORM[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
static const int OF_NORM[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
static const uint32_t LL_BASE[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40,
                                     48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
static const uint8_t LL_BITS[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9,
                                    10, 11, 12, 13, 14, 15, 16};
static const uint32_t ML_BASE_HI[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                        16387, 32771, 65539};
static const uint8_t ML_BITS_HI[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

// enc[s * size + x] for a distribution norm[n] of accuracy log `log`
static void fse_enc(const int *norm, int n, int log, uint16_t *enc) {
    const int size = 1 << log;
    int sym[64], high = size - 1;
    for (int s = 0; s < n; s++) if (norm[s] == -1) sym[high--] = s;
    const int step = (size >> 1) + (size >> 3) + 3;
    for (int s = 0, pos = 0; s < n; s++)
        for (int k = 0; k < norm[s]; k++) {
            sym[pos] = s;
            do pos = (pos + step) & (size - 1); while (pos > high);
        }
    int next[64];
    for (int s = 0; s < n; s++) next[s] = norm[s] == -1 ? 1 : norm[s];
    for (int u = 0; u < size; u++) {
        const int x = next[sym[u]]++;
        int hb = 0;
        while ((x >> (hb + 1)) != 0) hb++;
        const int nb = log - hb, baseline = (x << nb) - size;
        for (int y = baseline; y < baseline + (1 << nb); y++)
            enc[sym[u] * size + y] = (uint16_t)(u | nb << 6 | (y - baseline) << 9);
    }
}

void lz_fill_tables_host(void *dst) {
    LzTables t;
    memset(&t, 0, sizeof t);
    fse_enc(LL_NORM, 36, 6, &t.ll_enc[0][0]);
    fse_enc(ML_NORM, 53, 6, &t.ml_enc[0][0]);
    fse_enc(OF_NORM, 29, 5, &t.of_enc[0][0]);
    for (int c = 0; c < 36; c++) { t.ll_base[c] = LL_BASE[c]; t.ll_bits[c] = LL_BITS[c]; }
    for (int c = 0; c < 53; c++) {
        t.ml_base[c] = c < 32 ? c + 3 : ML_BASE_HI[c - 32];
        t.ml_bits[c] = c < 32 ? 0 : ML_BITS_HI[c - 32];
    }
    for (uint32_t v = 0, c = 0; v < 64; v++) { while (c + 1 < 36 && LL_BASE[c + 1] <= v) c++; t.ll_code[v] = (uint8_t)c; }
    for (uint32_t v = 0, c = 0; v < 128; v++) { while (c + 1 < 53 && t.ml_base[c + 1] <= v + 3) c++; t.ml_code[v] = (uint8_t)c; }
    memcpy(dst, &t, sizeof t);
}

}  // namespace pbsgpu
