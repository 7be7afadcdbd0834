// pbs_plus_b200/csrc/zent.cuh -- the constants that define K10's output bytes (zent.cu) and its launch interface.
// tests/zstd_ent_ref.py (LL_MAXLOG, OF_MAXLOG, ML_MAXLOG, MIN_LOG, HUF_MAXBITS, HUF_MAXSYMBOL) and tests/zstd_huf_ref.py
// (WEIGHT_MAXLOG, FSE_TREE_MAX) state the same values; DESIGN.md K10 has the tables the accuracy-log rule comes from.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pbsgpu {

constexpr int ENT_LL_MAXLOG = 9, ENT_OF_MAXLOG = 8, ENT_ML_MAXLOG = 9;   // the format's largest FSE accuracy logs
constexpr int ENT_MIN_LOG = 5;                                            // the smallest one a table description states
constexpr int ENT_HUF_MAXBITS = 11;       // longest Huffman code of the literals
constexpr int ENT_HUF_MAXSYMBOL = 128;    // the direct weight form lists at most 128 weights (the last one is implied)
constexpr int ENT_WEIGHT_MAXLOG = 6;      // the largest accuracy log of the FSE table of Huffman weights
constexpr int ENT_FSE_TREE_MAX = 127;     // the FSE weight form's header byte is its size, below 128

constexpr uint32_t ENT_SCRATCH = 2 * LZ_SLOT;   // per block of a pass: Huffman literals section, then the FSE bitstream

// Huffman code lengths of the symbols 0..nsym-1 with counts cnt[] (m >= 2 of them present), longest at most `limit`,
// built by one warp (K10's literals, K15's three codes): present symbols in (count, symbol) order; two-queue Huffman
// where each step joins the two smallest fronts, a leaf before a node of equal count, and a parent is made after its
// children; while the longest code is above `limit` the counts are halved, rounding up, and the code is built again.
// Writes hlen[] of the present symbols only and returns the longest length in every lane.  Scratch: hc[nsym],
// horder[m], hw[2m-1], hparent[2m-1], hdepth[2m-1]; *maxlen is a shared word.
template <typename Sym>
__device__ inline uint32_t huf_lengths(const uint32_t *cnt, uint32_t nsym, uint32_t m, uint32_t limit, uint32_t lane,
                                       uint32_t *hc, Sym *horder, uint32_t *hw, uint16_t *hparent, uint8_t *hdepth,
                                       uint8_t *hlen, uint32_t *maxlen) {
    for (uint32_t x = lane; x < nsym; x += 32) hc[x] = cnt[x];
    __syncwarp();
    for (;;) {
        for (uint32_t x = lane; x < nsym; x += 32) {
            const uint32_t c = hc[x];
            if (!c) continue;
            uint32_t r = 0;
            for (uint32_t y = 0; y < nsym; y++) { const uint32_t e = hc[y]; r += e && (e < c || (e == c && y < x)); }
            horder[r] = (Sym)x;
        }
        __syncwarp();
        if (lane == 0) {
            for (uint32_t k = 0; k < m; k++) hw[k] = hc[horder[k]];
            uint32_t i = 0, j = m, nxt = m;
            for (uint32_t k = 0; k + 1 < m; k++, nxt++) {
                uint32_t a, b;
                if (i < m && (j >= nxt || hw[i] <= hw[j])) a = i++; else a = j++;
                if (i < m && (j >= nxt || hw[i] <= hw[j])) b = i++; else b = j++;
                hw[nxt] = hw[a] + hw[b];
                hparent[a] = hparent[b] = (uint16_t)nxt;
            }
            hdepth[2 * m - 2] = 0;
            for (int k = 2 * (int)m - 3; k >= 0; k--) hdepth[k] = hdepth[hparent[k]] + 1;
            uint32_t mx = 0;
            for (uint32_t k = 0; k < m; k++) { hlen[horder[k]] = hdepth[k]; mx = max(mx, (uint32_t)hdepth[k]); }
            *maxlen = mx;
        }
        __syncwarp();
        if (*maxlen <= limit) break;
        for (uint32_t x = lane; x < nsym; x += 32) hc[x] = (hc[x] + 1) >> 1;   // a present symbol stays present
        __syncwarp();
    }
    return *maxlen;
}

// K10: after K9b, for blocks [first, first + nb) with K9a's literals (slot + 3) and sequences (seqs + (g - first) *
// LZ_MAX_SEQ): the entropy-coded Block_Content, which replaces K9b's in the slot (and info[g], same form) when it is
// smaller than both K9b's content and the block (size[g]).  scratch holds nb * ENT_SCRATCH bytes.  `full` (the _lzh
// encoder): Huffman literals whatever their largest value, with the FSE-compressed weight form of the tree where it is
// allowed and smaller than the direct one; the content is then never larger than with `full` off.
cudaError_t launch_ent_encode(const LzTables *tab, const uint32_t *size, uint64_t first, uint32_t nb, uint8_t *slots,
                              const uint64_t *seqs, const uint32_t *nseq, const uint32_t *nlit, uint32_t *info,
                              uint8_t *scratch, bool full, cudaStream_t st);

}  // namespace pbsgpu
