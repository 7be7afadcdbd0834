// pbs_plus_b200/csrc/zlz.cuh -- the constants that define K9's output bytes (zlz.cu), its launch interface, and the
// sequences writer K9b shares with K10.  tests/zstd_lz_ref.py (LZ_HBITS, LZ_TILE, LZ_MINMATCH) states the same
// values; DESIGN.md K9 has the table they come from.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pbsgpu {

constexpr int LZ_HBITS = 13;      // hash table of 2^13 positions
constexpr int LZ_TILE = 256;      // positions looked up before any of them is inserted
constexpr int LZ_MINMATCH = 4;    // shortest match

constexpr uint32_t LZ_SLOT = 128u * 1024u + 16u;         // per-block output slot: 3 bytes of room for the literals header
constexpr uint32_t LZ_MAX_SEQ = 128u * 1024u / LZ_MINMATCH;   // every sequence covers >= LZ_MINMATCH bytes of its block
constexpr uint32_t LZ_PASS_BLOCKS = 4096;                // blocks per pass: 1 GiB of sequence scratch

// The Predefined_Mode distributions of the LL, ML and OF codes (RFC 8878 3.1.1.3.2.2), accuracy logs 6, 6 and 5
constexpr int16_t PREDEF_LL_NORM[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1,
                                        1, 1, -1, -1, -1, -1};
constexpr int16_t PREDEF_ML_NORM[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                        1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
constexpr int16_t PREDEF_OF_NORM[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1,
                                        -1, -1};

// The Literals_Length / Match_Length codes (RFC 8878 3.1.1.3.2.1.1), read by K9b and K10.
struct SeqCodes {
    uint32_t ll_base[36], ml_base[53];   // Literals_Length / Match_Length baselines (Match_Length in bytes, >= 3)
    uint8_t ll_bits[36], ml_bits[53];
    uint8_t ll_code[64], ml_code[128];   // code of a literal length < 64 and of a match length - 3 < 128
};

// What both kernels read, built on the host (lz_fill_tables_host): the codes and the Predefined_Mode FSE tables
// (RFC 8878 3.1.1.3.2.2) of K9b in fse_ctable's form.
struct alignas(16) LzTables {
    SeqCodes codes;
    uint16_t ll_stab[64], of_stab[32], ml_stab[64];
    int32_t ll_dnb[36], ll_dfs[36], of_dnb[29], of_dfs[29], ml_dnb[53], ml_dfs[53];
};
static_assert(sizeof(LzTables) % 16 == 0, "copied to shared memory in 16-byte words");
void lz_fill_tables_host(void *dst);

// The encoder form of the FSE table of norm[0..nsym) at accuracy log `log` (zstd's FSE_buildCTable). The codes are
// spread over the states (RFC 8878 4.1.1; spread[] is scratch): a "less than 1" code (-1) takes one state at the top
// of the table, and the spread skips those states. stab lists the states of each code in state order, grouped by
// code. Per code, dnb gives the Number_of_Bits to write from a state X (kept as 2^log + state) and dfs the offset of
// the next state in stab (zstd's symbolTT); a -1 code has the transform of a code with one state.
// The code of every state of the FSE table of norm[0..nsym) at accuracy log `log` (RFC 8878 4.1.1), into spread[0, 2^log):
// a "less than 1" code (-1) takes one state at the top of the table, and the other codes are spread over the states
// below them.  The counts must sum to 2^log (the absolute value of a -1), as every valid table description does.  The
// encoder form (fse_ctable) and the decoder form (fse_dtable, zdec.cuh) are both built from it.
__host__ __device__ inline void fse_spread(const int16_t *norm, int nsym, int log, uint8_t *spread) {
    const int size = 1 << log, step = (size >> 1) + (size >> 3) + 3;
    int high = size - 1;
    for (int c = 0; c < nsym; c++) if (norm[c] == -1) spread[high--] = (uint8_t)c;
    for (int c = 0, pos = 0; c < nsym; c++)
        for (int k = 0; k < norm[c]; k++) {
            spread[pos] = (uint8_t)c;
            do pos = (pos + step) & (size - 1); while (pos > high);
        }
}

__host__ __device__ inline void fse_ctable(const int16_t *norm, int nsym, int log, uint8_t *spread, uint16_t *stab,
                                           int32_t *dnb, int32_t *dfs) {
    const int size = 1 << log;
    fse_spread(norm, nsym, log, spread);
    int32_t *next = dnb;   // the next free place of each code in stab, before dnb takes its final value
    for (int c = 0, cum = 0; c < nsym; c++) { next[c] = cum; cum += norm[c] == -1 ? 1 : norm[c]; }
    for (int u = 0; u < size; u++) stab[next[spread[u]]++] = (uint16_t)u;
    for (int c = 0; c < nsym; c++) {
        const int k = norm[c] == -1 ? 1 : norm[c], start = next[c] - k;
        if (k == 0) { dnb[c] = 0; dfs[c] = 0; continue; }
        if (k == 1) { dnb[c] = (log << 16) - size; dfs[c] = start - 1; continue; }
        int out = 1;   // log - floor(log2(k - 1)): (k - 1) << out lands in [size, 2 size)
        while (((k - 1) << out) < size) out++;
        dnb[c] = (out << 16) - (k << out);
        dfs[c] = start - k;
    }
}

// Raw_Literals_Block header size for nl literals (Size_Format 00 / 01 / 11)
__host__ __device__ inline uint32_t raw_lit_header_len(uint32_t nl) { return nl <= 31 ? 1 : nl <= 4095 ? 2 : 3; }

// Number_of_Sequences (1, 2 or 3 bytes) into out; returns its size
__device__ inline uint32_t seq_count_header(uint32_t n, uint8_t *out) {
    if (n < 128) { out[0] = (uint8_t)n; return 1; }
    if (n < 0x7F00) { out[0] = (uint8_t)((n >> 8) + 0x80); out[1] = (uint8_t)n; return 2; }
    out[0] = 0xFF; out[1] = (uint8_t)(n - 0x7F00); out[2] = (uint8_t)((n - 0x7F00) >> 8);
    return 3;
}

// LL / ML / OF code, value and Offset_Value of a packed K9a sequence
struct Seq {
    uint32_t ll, ml, ov, lc, mc, oc;
    __device__ Seq(uint64_t v, const SeqCodes &c) {
        ll = (uint32_t)(v & 0xFFFFF); ml = (uint32_t)((v >> 20) & 0xFFFFF); ov = (uint32_t)(v >> 40) + 3;
        lc = ll < 64 ? c.ll_code[ll] : 31 - __clz(ll) + 19;
        mc = ml - 3 < 128 ? c.ml_code[ml - 3] : 31 - __clz(ml - 3) + 36;
        oc = 31 - __clz(ov);
    }
};

// Bits are appended LSB first; bytes at or beyond LZ_SLOT are counted but not stored (such a block stays raw).
struct LzBits {
    uint8_t *slot;
    uint32_t q;
    uint64_t acc = 0;
    uint32_t n = 0;
    __device__ void byte(uint32_t v) { if (q < LZ_SLOT) slot[q] = (uint8_t)v; q++; }
    __device__ void add(uint32_t v, uint32_t nb) {
        acc |= (uint64_t)v << n;
        n += nb;
        while (n >= 8) { byte((uint32_t)acc); acc >>= 8; n -= 8; }
    }
};

// One FSE table in fse_ctable's form
struct FseCTable {
    const uint16_t *stab;
    const int32_t *dnb, *dfs;
    uint32_t log;
    // from state x (2^log + state): the state in which the decoder reads code c and then goes to x; the bits it reads
    // to get there go to w when `write` is set
    __device__ __forceinline__ uint32_t step(uint32_t x, uint32_t c, LzBits &w, bool write) const {
        const uint32_t nb = (uint32_t)((int)x + dnb[c]) >> 16;
        if (write) w.add(x & ((1u << nb) - 1), nb);
        return (1u << log) + stab[(int)(x >> nb) + dfs[c]];
    }
};

// The FSE bitstream of a Sequences_Section (RFC 8878 3.1.1.3.2.2) of n >= 1 packed K9a sequences, tables t = LL, OF,
// ML, with its end mark and final partial byte. Written forward, read backward: the last sequence's extra bits (LL, ML,
// OF) come first, then per earlier sequence the state bits (OF, ML, LL) that lead to its successor's states and its
// extra bits, then the first sequence's states (ML, OF, LL) and the end mark. The last sequence starts in the state
// from which the decoder goes to state 0, so its state bits are zeros and are not written.
__device__ __forceinline__ void seq_bitstream(const uint64_t *sq, uint32_t n, const SeqCodes &sc, const FseCTable (&t)[3],
                                              LzBits &w) {
    uint32_t X[3] = {1u << t[0].log, 1u << t[1].log, 1u << t[2].log};
    for (uint32_t k = n; k-- > 0;) {
        const Seq q(sq[k], sc);
        const bool wr = k + 1 < n;
        X[1] = t[1].step(X[1], q.oc, w, wr); X[2] = t[2].step(X[2], q.mc, w, wr); X[0] = t[0].step(X[0], q.lc, w, wr);
        w.add(q.ll - sc.ll_base[q.lc], sc.ll_bits[q.lc]);
        w.add(q.ml - sc.ml_base[q.mc], sc.ml_bits[q.mc]);
        w.add(q.ov - (1u << q.oc), q.oc);
    }
    w.add(X[2] - (1u << t[2].log), t[2].log); w.add(X[1] - (1u << t[1].log), t[1].log);
    w.add(X[0] - (1u << t[0].log), t[0].log); w.add(1, 1);
    if (w.n) w.byte((uint32_t)w.acc);
}

// K9a: blocks [first, first + nb) of the list (src[], size[]); literals to slots + g * LZ_SLOT + 3, sequences to
// seqs + (g - first) * LZ_MAX_SEQ, counts to nseq[g] / nlit[g].
cudaError_t launch_lz_parse(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint64_t first, uint32_t nb,
                            uint8_t *slots, uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st);
// K9a with long spans (the _lzl span parse): block g's spans are spans[span_first[g - sbase] .. span_first[g - sbase + 1]),
// each start | length << 20 | offset << 40 (start and length inside the block, length >= LZ_MINMATCH), in order.
cudaError_t launch_lz_parse_spans(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint64_t first, uint32_t nb,
                                  uint8_t *slots, uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, const uint64_t *spans,
                                  const uint32_t *span_first, uint64_t sbase, cudaStream_t st);
// K9a with the Deflate limits of deflate.cuh (K15's parse): blocks [0, nb) of (src[], size[]), outputs as launch_lz_parse's
// with first = 0.
cudaError_t launch_lz_parse_deflate(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint32_t nb, uint8_t *slots,
                                    uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st);
// K9b: the Block_Content of those blocks in their slots; info[g] = content size | (offset of the content in the slot) << 30.
// A size >= the block's size means the block stays raw (the slot then holds only its first LZ_SLOT bytes).
cudaError_t launch_lz_encode(const LzTables *tab, uint64_t first, uint32_t nb, uint8_t *slots, const uint64_t *seqs,
                             const uint32_t *nseq, const uint32_t *nlit, uint32_t *info, cudaStream_t st);

}  // namespace pbsgpu
