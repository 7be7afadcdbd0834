// pbs_plus_b200/csrc/zldm.cuh -- the constants that define K12's output bytes (zldm.cu, the long-distance matches of
// _lzl) and its launch interface.  tests/zstd_ldm_ref.py (LDM_RATE, LDM_MINMATCH, LDM_MAXDIST, LDM_SEED) states the same
// values; DESIGN.md K12 has the sweep LDM_RATE comes from.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pbsgpu {

constexpr int LDM_RATE = 7;                          // anchor: the top 7 bits of the gear hash are zero (1 in 128)
constexpr uint32_t LDM_WINDOW = 64;                  // bytes hashed per anchor
constexpr uint32_t LDM_MINMATCH = 64;                // shortest kept long match
constexpr uint32_t LDM_MAXDIST = (1u << 24) - 4;     // largest offset: K9's packed sequences keep it in 24 bits
constexpr uint64_t LDM_SEED = 0;                     // splitmix64 seed of the gear table (no constant run has an anchor)

constexpr uint32_t LDM_SPAN = 2048;                        // anchor-scan positions per thread (+ 63 bytes of warm-up)
constexpr uint64_t LDM_PASS_BYTES = 64ull << 20;           // chunk bytes per pass (a longer chunk is a pass of its own)
constexpr uint32_t LDM_PASS_CHUNKS = (1u << 24) - 2;       // chunks per pass: the chunk index takes 24 bits of a key
constexpr uint64_t LDM_M40 = (1ull << 40) - 1;

// anchor-scan spans of a chunk of len bytes: positions [63, len) in runs of LDM_SPAN
__host__ __device__ inline uint64_t ldm_spans(uint64_t len) {
    return len >= LDM_WINDOW ? (len - (LDM_WINDOW - 1) + LDM_SPAN - 1) / LDM_SPAN : 0;
}

// One pass: chunks [c0, c1) of the call's list (off[], len[]), whose anchor-scan spans are [span_first[c0],
// span_first[c1]); vfirst[i] = bytes of the chunks before i (a pass numbers its bytes from vfirst[c0]).
struct LdmArgs {
    const uint8_t *base;
    const uint64_t *off, *len, *span_first, *vfirst;
    uint32_t c0, c1;
    uint64_t s0, s1;
};

// K12a (count only): the number of anchors of the pass, added to *total
cudaError_t launch_ldm_count(const LdmArgs &a, unsigned long long *total, cudaStream_t st);
// scratch of a pass with `spans` anchor-scan spans and `anchors` anchors
size_t ldm_scratch_bytes(uint64_t spans, uint64_t anchors);
// K12 over one pass of `anchors` anchors (launch_ldm_count's total): the kept long matches of each chunk, at
// (*key)[k] = chunk in the pass << 40 | start, (*val)[k] = offset << 40 | end (chunk positions), k < *n_kept (device; in
// no particular order).  The three pointers point into scratch.
cudaError_t launch_ldm_matches(const LdmArgs &a, uint64_t anchors, void *scratch, uint64_t **key, uint64_t **val,
                               uint32_t **n_kept, cudaStream_t st);

}  // namespace pbsgpu
