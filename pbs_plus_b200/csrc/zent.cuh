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

// K10: after K9b, for blocks [first, first + nb) with K9a's literals (slot + 3) and sequences (seqs + (g - first) *
// LZ_MAX_SEQ): the entropy-coded Block_Content, which replaces K9b's in the slot (and info[g], same form) when it is
// smaller than both K9b's content and the block (size[g]).  scratch holds nb * ENT_SCRATCH bytes.  `full` (the _lzh
// encoder): Huffman literals whatever their largest value, with the FSE-compressed weight form of the tree where it is
// allowed and smaller than the direct one; the content is then never larger than with `full` off.
cudaError_t launch_ent_encode(const LzTables *tab, const uint32_t *size, uint64_t first, uint32_t nb, uint8_t *slots,
                              const uint64_t *seqs, const uint32_t *nseq, const uint32_t *nlit, uint32_t *info,
                              uint8_t *scratch, bool full, cudaStream_t st);

}  // namespace pbsgpu
