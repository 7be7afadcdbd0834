// pbs_plus_b200/csrc/zlz.cuh -- the constants that define K9's output bytes (zlz.cu) and its launch interface.
// tests/zstd_lz_ref.py (LZ_HBITS, LZ_TILE, LZ_MINMATCH) states the same values; DESIGN.md K9 has the table they come from.
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

// Predefined_Mode FSE tables (RFC 8878 3.1.1.3.2.2) in the encoder's form, built on the host (lz_fill_tables_host).
// xx_enc[s][x]: the state to be in when the decoder must read symbol s and then go to state x, packed as
// state | Number_of_Bits << 6 | (x - Baseline) << 9.
struct LzTables {
    uint16_t ll_enc[36][64], ml_enc[53][64], of_enc[29][32];
    uint32_t ll_base[36], ml_base[53];   // Literals_Length / Match_Length baselines (Match_Length in bytes, >= 3)
    uint8_t ll_bits[36], ml_bits[53];
    uint8_t ll_code[64], ml_code[128];   // code of a literal length < 64 and of a match length - 3 < 128
    uint8_t pad[3];
};
static_assert(sizeof(LzTables) % 16 == 0, "copied to shared memory in 16-byte words");
void lz_fill_tables_host(void *dst);

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

// K9a: blocks [first, first + nb) of the list (src[], size[]); literals to slots + g * LZ_SLOT + 3, sequences to
// seqs + (g - first) * LZ_MAX_SEQ, counts to nseq[g] / nlit[g].
cudaError_t launch_lz_parse(const uint8_t *base, const uint64_t *src, const uint32_t *size, uint64_t first, uint32_t nb,
                            uint8_t *slots, uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st);
// K9b: the Block_Content of those blocks in their slots; info[g] = content size | (offset of the content in the slot) << 30.
// A size >= the block's size means the block stays raw (the slot then holds only its first LZ_SLOT bytes).
cudaError_t launch_lz_encode(const LzTables *tab, uint64_t first, uint32_t nb, uint8_t *slots, const uint64_t *seqs,
                             const uint32_t *nseq, const uint32_t *nlit, uint32_t *info, cudaStream_t st);

}  // namespace pbsgpu
