// f3: the LZ77 match stage and Predefined_Mode sequences of compressed DataBlobs (K9, sm_90a).
//
// Every 128 KiB block of a chunk that is not one repeated byte (K8a decides that) becomes a zstd Compressed_Block
// (RFC 8878 3.1.1.3): a greedy LZ77 parse inside the block, Raw_Literals and a sequences section whose three FSE tables
// are the predefined ones.  The host (capi_blob.cu, zstd_frames) keeps that block when it is smaller than the raw one.
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
//                     front of the literals, the sequences header, the modes byte and the bitstream (seq_bitstream),
//                     behind them in the slot.  The tables sit in shared memory; the 32 blocks of a warp run in step.
#include "internal.cuh"

#include <cstring>

namespace pbsgpu {

constexpr int LZ_THREADS = 256;
static_assert(LZ_TILE == LZ_THREADS, "one position per thread per tile");

__device__ __forceinline__ uint32_t lz_key(const uint8_t *p) {
    return (uint32_t)__ldg(p) | (uint32_t)__ldg(p + 1) << 8 | (uint32_t)__ldg(p + 2) << 16 | (uint32_t)__ldg(p + 3) << 24;
}

// SPANS (the _lzl span parse): block g also has the long spans spans[span_first[g - sbase] .. span_first[g - sbase + 1]),
// packed start | length << 20 | offset << 40 and in order.  A span is taken where it starts and the parse jumps past
// it; a match is cut at the next span's start and kept only while it is still >= LZ_MINMATCH long.
// DEFLATE (K15's parse, deflate.cuh): a candidate counts only at distance <= DEFLATE_WINDOW, and a match is cut at
// DEFLATE_MAX_MATCH; the parse resumes behind the cut match.
template <bool SPANS, bool DEFLATE = false>
__global__ void __launch_bounds__(LZ_THREADS) k_lz_parse(const uint8_t *base, const uint64_t *src, const uint32_t *size,
                                                         uint64_t first, uint8_t *slots, uint64_t *seqs, uint32_t *nseq,
                                                         uint32_t *nlit, const uint64_t *spans, const uint32_t *span_first,
                                                         uint64_t sbase) {
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
    uint32_t sj = 0, send = 0, ss = ~0u, sl = 0, sd = 0;   // SPANS: the next span (start ss; ~0u: none left)
    auto next_span = [&] {
        ss = ~0u;
        if (sj < send) { const uint64_t v = spans[sj]; ss = v & 0xFFFFF; sl = (v >> 20) & 0xFFFFF; sd = (uint32_t)(v >> 40); }
    };
    if (SPANS) { sj = span_first[g - sbase]; send = span_first[g - sbase + 1]; next_span(); }
    for (uint32_t t0 = 0; t0 < nk; t0 += LZ_TILE) {
        const uint32_t tend = min(t0 + LZ_TILE, nk);
        const uint32_t i = t0 + threadIdx.x;
        uint32_t h = 0;
        if (i < tend) {
            const uint32_t key = lz_key(p + i);
            h = (key * 0x9E3779B1u) >> (32 - LZ_HBITS);
            const int c = table[h];
            bool m = c >= 0 && (!DEFLATE || i - (uint32_t)c <= DEFLATE_WINDOW) && lz_key(p + c) == key;
#pragma unroll
            for (int e = 4; e < LZ_MINMATCH; e++) m = m && i + e < S && __ldg(p + c + e) == __ldg(p + i + e);
            cand[threadIdx.x] = m ? c : -1;
        }
        __syncthreads();
        if (i < tend) atomicMax(&table[h], (int)i);
        if (parser) {
            while (pos < tend) {
                if (SPANS && pos == ss) {
                    if (lane == 0) sq[ns] = (uint64_t)(ss - run) | (uint64_t)sl << 20 | (uint64_t)sd << 40;
                    ns++;
                    pos = run = ss + sl;
                    sj++;
                    next_span();
                    continue;
                }
                const uint32_t lim = SPANS ? min(tend, ss) : tend;
                const uint32_t q = pos + lane;
                const uint32_t hits = __ballot_sync(~0u, q < lim && cand[q - t0] >= 0);
                const uint32_t m = hits ? pos + __ffs(hits) - 1 : min(pos + 32, lim);
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
                    if (DEFLATE && L >= DEFLATE_MAX_MATCH) break;
                }
                if (DEFLATE) L = min(L, DEFLATE_MAX_MATCH);
                if (SPANS && ss != ~0u) {
                    L = min(L, ss - m);
                    if (L < LZ_MINMATCH) {   // too short once cut: m is a literal
                        if (lane == 0) lit[nl] = __ldg(p + m);
                        nl++;
                        pos = m + 1;
                        continue;
                    }
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
    k_lz_parse<false><<<nb, LZ_THREADS, 0, st>>>(base, src, size, first, slots, seqs, nseq, nlit, nullptr, nullptr, 0);
    return cudaGetLastError();
}

cudaError_t launch_lz_parse_spans(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint64_t first, uint32_t nb,
                                  uint8_t *slots, uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, const uint64_t *spans,
                                  const uint32_t *span_first, uint64_t sbase, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    k_lz_parse<true><<<nb, LZ_THREADS, 0, st>>>(base, src, size, first, slots, seqs, nseq, nlit, spans, span_first, sbase);
    return cudaGetLastError();
}

cudaError_t launch_lz_parse_deflate(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint32_t nb, uint8_t *slots,
                                    uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    k_lz_parse<false, true><<<nb, LZ_THREADS, 0, st>>>(base, src, size, 0, slots, seqs, nseq, nlit, nullptr, nullptr, 0);
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
    const uint32_t n = nseq[g], nl = nlit[g], hl = raw_lit_header_len(nl);
    LzBits w{slots + g * LZ_SLOT, 3 - hl};
    if (hl == 1) w.byte(nl << 3);
    else if (hl == 2) { w.byte((nl << 4) | 0x4); w.byte(nl >> 4); }
    else { w.byte((nl << 4) | 0xC); w.byte(nl >> 4); w.byte(nl >> 12); }
    w.q = 3 + nl;
    w.q += seq_count_header(n, w.slot + w.q);   // within the slot: 3 + nl + 3 <= LZ_SLOT
    if (n) {
        w.byte(0);   // Symbol_Compression_Modes: all Predefined_Mode
        const FseCTable t[3] = {{T.ll_stab, T.ll_dnb, T.ll_dfs, 6}, {T.of_stab, T.of_dnb, T.of_dfs, 5},
                                {T.ml_stab, T.ml_dnb, T.ml_dfs, 6}};
        seq_bitstream(seqs + (uint64_t)b * LZ_MAX_SEQ, n, T.codes, t, w);
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
static const uint32_t LL_BASE[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40,
                                     48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
static const uint8_t LL_BITS[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9,
                                    10, 11, 12, 13, 14, 15, 16};
static const uint32_t ML_BASE_HI[21] = {35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                        16387, 32771, 65539};
static const uint8_t ML_BITS_HI[21] = {1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

void lz_fill_tables_host(void *dst) {
    LzTables t;
    memset(&t, 0, sizeof t);
    uint8_t spread[64];
    fse_ctable(PREDEF_LL_NORM, 36, 6, spread, t.ll_stab, t.ll_dnb, t.ll_dfs);
    fse_ctable(PREDEF_OF_NORM, 29, 5, spread, t.of_stab, t.of_dnb, t.of_dfs);
    fse_ctable(PREDEF_ML_NORM, 53, 6, spread, t.ml_stab, t.ml_dnb, t.ml_dfs);
    SeqCodes &s = t.codes;
    for (int c = 0; c < 36; c++) { s.ll_base[c] = LL_BASE[c]; s.ll_bits[c] = LL_BITS[c]; }
    for (int c = 0; c < 53; c++) {
        s.ml_base[c] = c < 32 ? c + 3 : ML_BASE_HI[c - 32];
        s.ml_bits[c] = c < 32 ? 0 : ML_BITS_HI[c - 32];
    }
    for (uint32_t v = 0, c = 0; v < 64; v++) { while (c + 1 < 36 && LL_BASE[c + 1] <= v) c++; s.ll_code[v] = (uint8_t)c; }
    for (uint32_t v = 0, c = 0; v < 128; v++) { while (c + 1 < 53 && s.ml_base[c + 1] <= v + 3) c++; s.ml_code[v] = (uint8_t)c; }
    memcpy(dst, &t, sizeof t);
}

}  // namespace pbsgpu
