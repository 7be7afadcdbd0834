// pbs_plus_b200/csrc/zdec.cuh -- K13 (zdec.cu): the zstd decoder of pbsgpu_blob_decode_batch, its limits and launch
// interface.  DESIGN.md K13 states the accepted format and the stages.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pbsgpu {

constexpr uint32_t ZDEC_LIT_SLOT = 128u * 1024u;          // per blob of a pass: the literals of one block
constexpr uint64_t ZDEC_PASS_BYTES = 2ull << 30;          // decoded bytes per pass of whole blobs (or one longer blob)
constexpr uint32_t ZDEC_PASS_BLOBS = 4096;                // blobs per pass: 512 MiB of literal scratch

// An FSE decoding table entry: the code of the state, the bits to read and the baseline of the next state
__host__ __device__ inline uint32_t fse_dentry(uint32_t sym, uint32_t nb, uint32_t base) { return sym | nb << 8 | base << 16; }

// The decoder form of the FSE table of norm[0..nsym) at accuracy log `log` (RFC 8878 4.1.1; zstd's FSE_buildDTable):
// dt[state] for the 2^log states; spread[] and next[nsym] are scratch.
__host__ __device__ inline void fse_dtable(const int16_t *norm, int nsym, int log, uint8_t *spread, uint16_t *next,
                                           uint32_t *dt) {
    const int size = 1 << log;
    fse_spread(norm, nsym, log, spread);
    for (int c = 0; c < nsym; c++) next[c] = (uint16_t)(norm[c] == -1 ? 1 : norm[c] > 0 ? norm[c] : 0);
    for (int u = 0; u < size; u++) {
        const uint32_t c = spread[u], x = next[c]++;
        uint32_t hb = 0;
        while ((x >> hb) > 1) hb++;
        const uint32_t nb = (uint32_t)log - hb;
        dt[u] = fse_dentry(c, nb, (x << nb) - (uint32_t)size);
    }
}

// What K13 reads besides the blobs, built on the host: the LL / ML codes and the Predefined_Mode tables in fse_dtable's form
struct alignas(16) ZdecTables {
    SeqCodes codes;
    uint32_t ll_dt[64], of_dt[32], ml_dt[64];
};
void zdec_fill_tables_host(void *dst);

// One blob of a pass: its bytes at base + src (len bytes), its chunk to dst (cap bytes: the expected chunk size)
struct ZdecBlob {
    uint64_t src, len;
    uint64_t dst, cap;
};
// K13: blobs b[0, nb) with the CRC-32 of their payloads crc[0, nb) (K6); status[k] = a PBSGPU_DEC_* value, PBSGPU_DEC_OK
// when the chunk was decoded to dst with the expected size and every content checksum matched.  lits holds
// nb * ZDEC_LIT_SLOT bytes of scratch.
cudaError_t launch_zdec(const uint8_t *base, const ZdecBlob *b, const uint32_t *crc, uint32_t nb, const ZdecTables *tab,
                        uint8_t *lits, int32_t *status, cudaStream_t st);

// Encrypted blobs (pbsgpu_blob_decode_batch_enc).  The host reads each blob's header {magic, crc, iv, tag}: from a
// device base, launch_blob_heads gathers the first ZDEC_HEAD bytes of blob i (zero-filled past its end) to
// heads + ZDEC_HEAD * i for one D2H copy.  A decrypted payload is laid out in the plaintext stage as a plain blob K13
// reads: launch_stage_heads writes head[k] (16 bytes: 4 of padding, the 12-byte plain header) to stage + at[k] (16 B
// aligned), and the plaintext follows at stage + at[k] + 16.
constexpr uint32_t ZDEC_HEAD = 44;
cudaError_t launch_blob_heads(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint32_t n, uint8_t *heads,
                              cudaStream_t st);
cudaError_t launch_stage_heads(uint8_t *stage, const uint64_t *at, const void *head, uint32_t n, cudaStream_t st);

}  // namespace pbsgpu
