// pbs_plus_b200/csrc/deflate.cuh -- the constants that define the raw Deflate streams (RFC 1951) of
// pbsgpu_deflate_batch (K9a's DEFLATE parse in zlz.cu, K15 in deflate.cu) and K15's launch interface.
// tests/deflate_ref.py states the same values and the format they define; DESIGN.md K15 describes it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pbsgpu {

constexpr uint32_t DEFLATE_SEGMENT = 128u * 1024u;   // bytes per independently coded segment (K9a's block)
constexpr uint32_t DEFLATE_WINDOW = 32768;           // largest match distance
constexpr uint32_t DEFLATE_MAX_MATCH = 258;          // longest match
constexpr uint32_t DEFLATE_STORED_MAX = 65535;       // bytes per stored block
constexpr uint32_t DEFLATE_MAXBITS = 15;             // longest lit/len and distance code
constexpr uint32_t DEFLATE_CL_MAXBITS = 7;           // longest code-length code
// a segment's output is never larger than its stored form: S + 5 bytes per stored block, at most 3 blocks
constexpr uint32_t DEFLATE_SLOT = DEFLATE_SEGMENT + 32;
constexpr uint32_t DEFLATE_PASS_SEGS = 4096;         // segments per pass: 1 GiB of sequence scratch, 512 MiB of output

// K15: segments [0, nb) of (src[], size[]), parsed by launch_lz_parse_deflate into lits (+ g * LZ_SLOT + 3), seqs
// (+ g * LZ_MAX_SEQ, rewritten in place) and nseq[] / nlit[]: each segment's Deflate blocks into out + g * DEFLATE_SLOT,
// out_len[g] bytes.  final[g]: the segment ends its stream (BFINAL); otherwise a fixed or dynamic form is followed by
// an empty stored block, so every segment ends byte-aligned.  size[g] >= 1.
cudaError_t launch_deflate_encode(const uint8_t *base, const uint64_t *src, const uint32_t *size, const uint8_t *final_,
                                  uint32_t nb, const uint8_t *lits, uint64_t *seqs, const uint32_t *nseq,
                                  const uint32_t *nlit, uint8_t *out, uint32_t *out_len, cudaStream_t st);

}  // namespace pbsgpu
