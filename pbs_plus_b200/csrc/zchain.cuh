// pbs_plus_b200/csrc/zchain.cuh -- the constants that define K16's output bytes (zchain.cu, the hash-chain match search
// and lazy parse of _lzc) and its launch interface.  tests/zstd_chain_ref.py (CH_MINMATCH, CH_DEPTH, CH_LAZY, CH_MARGIN,
// CH_MAXDIST) states the same values; DESIGN.md K16 has the table they come from.  The DEFLATE instantiation (the parse
// of pbsgpu_deflate_batch_lzc) has constants of its own, DCH_*: tests/deflate_chain_ref.py states them, DESIGN.md K16d
// has their sweep.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pbsgpu {

constexpr uint32_t CH_MINMATCH = 4;               // chain key: 4 bytes, the shortest match
constexpr uint32_t CH_DEPTH = 16;                 // chain entries searched per position
constexpr uint32_t CH_LAZY = 2;                   // positions the parse may move on from a match
constexpr int CH_MARGIN = 4;                      // gain a later match must exceed the current one's by
constexpr uint32_t CH_MAXDIST = (1u << 24) - 4;   // largest offset: K9's packed sequences keep it in 24 bits

constexpr uint32_t CH_CAP = 32;                   // K16b extends each candidate this far; beyond, K16c searches again
constexpr uint64_t CH_PASS_BYTES = 128ull << 20;  // chunk bytes per pass (a longer chunk is a pass of its own)

// Deflate (window 32768 and matches of at most 258 bytes, deflate.cuh): every 128 KiB segment is one chunk of one block
constexpr uint32_t DCH_MINMATCH = 3;              // chain key: 3 bytes, the shortest match
constexpr uint32_t DCH_DEPTH = 32;                // chain entries searched per position
constexpr uint32_t DCH_LAZY = 2;                  // positions the parse may move on from a match
constexpr int DCH_MARGIN = 4;                     // gain a later match must exceed the current one's by
constexpr uint32_t DCH_PASS_SEGS = 1024;          // segments per pass: 128 MiB of positions, about 3.5 GiB of scratch

// One pass: chunks [c0, c1) of the call's list (off[], len[]); vfirst[i] = bytes of the chunks before i, so position x
// of chunk i is pass position vfirst[i] - vfirst[c0] + x (< 2^32).  Its blocks that are not constant are [z0, z1) of the
// match stage's list (zsrc[], zsize[], as K9a's), and block z starts at pass position vpos[z] - vfirst[c0].  n: the
// pass's positions, vfirst[c1] - vfirst[c0].
struct ChainArgs {
    const uint8_t *base;
    const uint64_t *off, *len, *vfirst;
    uint32_t c0, c1;
    uint64_t n, vbase;   // vbase = vfirst[c0]
    const uint64_t *zsrc, *vpos;
    const uint32_t *zsize;
    uint64_t z0, z1;
};

// scratch of a pass of n positions
size_t chain_scratch_bytes(uint64_t n);
// K16a (prev of every position of the pass) and K16b (best of every position of its blocks) into scratch.  deflate: the
// DEFLATE instantiation, over a pass whose chunks are its blocks (c0 = z0, c1 = z1).
cudaError_t launch_chain_search(const ChainArgs &a, void *scratch, cudaStream_t st, bool deflate = false);
// K16c: the lazy parse of blocks [first, first + nb) of the pass (z0 <= first, first + nb <= z1, nb <= LZ_PASS_BLOCKS),
// from launch_chain_search's scratch; outputs as launch_lz_parse's.  deflate: as launch_lz_parse_deflate's (slots,
// nseq[] and nlit[] indexed from first, so K15 reads them), at most LZ_MAX_SEQ sequences per block.
cudaError_t launch_chain_parse(const ChainArgs &a, const void *scratch, uint64_t first, uint32_t nb, uint8_t *slots,
                               uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st, bool deflate = false);

}  // namespace pbsgpu
