// pbs_plus_b200/csrc/digestset.cu -- K4: known-digest set (insert / probe), device resident.
//
// Replaces the known-chunk bookkeeping of the reference's dedup session (seeded from the
// previous snapshot: backupproxy.PreviousBackupRef, reference internal/pxarmount/commit.go:
// 286-294, origPayloadIdx commit.go:324-329; "Only new chunks are uploaded",
// docs/pxar-mount.md:105).  Semantics = an exact set of 32-byte digests; a batch is
// processed in index order: hit[i] = digest i was in the set before the call OR equals
// some digest j < i of the same call.
//
// Deterministic and race free by construction:
//   1. sort (tag = first 8 digest bytes, index) with a stable radix sort (host calls CUB);
//   2. k_set_process: the first element of every run of equal digests is the
//      representative; later ones are hits.  Representatives probe the (quiescent) open-
//      addressing table with a full 32-byte compare; missing ones are inserted with a CAS
//      on the tag word -- all representatives are distinct digests, so a claimed slot is
//      never "maybe mine" and nobody reads half-written keys.
// The table never exceeds 50 % load (host grows + rehashes).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "device.cuh"
#include "internal.cuh"

namespace pbsgpu {

__device__ __forceinline__ uint64_t tag_of(const uint64_t *d) { uint64_t t = d[0]; return t ? t : 1ull; }
__device__ __forceinline__ uint64_t slot_hash(uint64_t t) {   // digests are uniform already; mix anyway (adversarial tags)
    t ^= t >> 33; t *= 0xff51afd7ed558ccdULL; t ^= t >> 33;
    return t;
}
__device__ __forceinline__ bool eq32(const uint64_t *a, const uint64_t *b) {
    return a[0] == b[0] && a[1] == b[1] && a[2] == b[2] && a[3] == b[3];
}

// The element count is *n_dev when n_dev is set (K4 as part of a batch job: the job's chunk count is only known on the
// device) and `cap` otherwise; `cap` bounds every launch.  Entries at index >= n get the all-ones tag and sort behind the
// real ones (a real digest whose first 8 bytes are all ones still works: the sort is stable, so it stays in front of the
// padding and padding threads return at once).

__global__ void k_set_make_keys(const uint8_t *d32, const unsigned long long *n_dev, uint64_t cap, uint64_t *tag, uint32_t *idx) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    tag[i] = i < live_count(n_dev ? *n_dev : cap, cap) ? tag_of((const uint64_t *)(d32 + i * 32)) : ~0ull;
    idx[i] = (uint32_t)i;
}
cudaError_t launch_set_make_keys(const uint8_t *d32, const unsigned long long *n_dev, uint64_t cap, uint64_t *tag, uint32_t *idx,
                                 cudaStream_t st) {
    if (!cap) return cudaSuccess;
    k_set_make_keys<<<(unsigned)((cap + 255) / 256), 256, 0, st>>>(d32, n_dev, cap, tag, idx);
    return cudaGetLastError();
}

// phase 0: mark in-batch duplicates + probe representatives.  phase 1: insert missing representatives.
// `guard` (optional): candidate counter of the job; when it exceeds guard_max the job's chunk list is truncated and will be
// recomputed, so this pass must not touch the table.
template <int PHASE>
__global__ void k_set_process(SetTable t, const uint8_t *d32, const uint64_t *tag_sorted, const uint32_t *idx_sorted,
                              const unsigned long long *n_dev, uint64_t cap, const unsigned long long *guard, uint64_t guard_max,
                              int do_insert, uint8_t *hit, uint8_t *is_rep_miss, unsigned long long *n_new) {
    uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= live_count(n_dev ? *n_dev : cap, cap)) return;   // the n real entries are the first n after the stable sort
    if (guard && *guard > guard_max) { if (PHASE == 0 && hit) hit[idx_sorted[j]] = 0; return; }
    const uint32_t i = idx_sorted[j];
    const uint64_t *d = (const uint64_t *)(d32 + (uint64_t)i * 32);
    const uint64_t tag = tag_sorted[j];
    if (PHASE == 0) {
        // representative = first (lowest index: the sort is stable) of its equal-digest run
        // (pure probe: plain membership, every element looks itself up)
        bool dup = false;
        if (do_insert && j > 0 && tag_sorted[j - 1] == tag) {
            // equal tags are adjacent; normally equal digests too.  Walk back over the tag run only while
            // digests differ (a 64-bit tag collision between distinct digests -- practically never).
            for (uint64_t k = j; k > 0 && tag_sorted[k - 1] == tag; k--) {
                if (eq32(d, (const uint64_t *)(d32 + (uint64_t)idx_sorted[k - 1] * 32))) { dup = true; break; }
            }
        }
        uint8_t h = 1, miss = 0;
        if (!dup) {
            h = 0;
            uint64_t slot = slot_hash(tag) & (t.cap - 1);
            for (;;) {
                uint64_t cur = t.tags[slot];
                if (cur == 0) break;
                if (cur == tag && eq32(d, t.keys + slot * 4)) { h = 1; break; }
                slot = (slot + 1) & (t.cap - 1);
            }
            miss = !h;
        }
        if (hit) hit[i] = h;
        is_rep_miss[j] = miss;
    } else {
        if (!is_rep_miss[j]) return;
        uint64_t slot = slot_hash(tag) & (t.cap - 1);
        for (;;) {
            unsigned long long cur = atomicCAS((unsigned long long *)&t.tags[slot], 0ull, (unsigned long long)tag);
            if (cur == 0) {   // claimed: nobody else reads keys[slot] during this kernel
                uint64_t *k = t.keys + slot * 4;
                k[0] = d[0]; k[1] = d[1]; k[2] = d[2]; k[3] = d[3];
                atomicAdd(n_new, 1ull);
                break;
            }
            slot = (slot + 1) & (t.cap - 1);   // occupied by a different digest (possibly same tag)
        }
    }
}

cudaError_t launch_set_mark_probe_insert(SetTable t, const uint8_t *d32, const uint64_t *tag_sorted, const uint32_t *idx_sorted,
                                         const unsigned long long *n_dev, uint64_t cap, const unsigned long long *guard,
                                         uint64_t guard_max, int do_insert, uint8_t *hit, uint8_t *is_rep_miss /*[cap] scratch*/,
                                         unsigned long long *n_new, cudaStream_t st) {
    if (!cap) return cudaSuccess;
    unsigned blocks = (unsigned)((cap + 255) / 256);
    k_set_process<0><<<blocks, 256, 0, st>>>(t, d32, tag_sorted, idx_sorted, n_dev, cap, guard, guard_max, do_insert, hit, is_rep_miss, n_new);
    if (do_insert)
        k_set_process<1><<<blocks, 256, 0, st>>>(t, d32, tag_sorted, idx_sorted, n_dev, cap, guard, guard_max, do_insert, hit, is_rep_miss, n_new);
    return cudaGetLastError();
}

__global__ void k_set_rehash(SetTable from, SetTable to) {
    uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= from.cap) return;
    uint64_t tag = from.tags[s];
    if (!tag) return;
    const uint64_t *d = from.keys + s * 4;
    uint64_t slot = slot_hash(tag) & (to.cap - 1);
    for (;;) {
        unsigned long long cur = atomicCAS((unsigned long long *)&to.tags[slot], 0ull, (unsigned long long)tag);
        if (cur == 0) { uint64_t *k = to.keys + slot * 4; k[0] = d[0]; k[1] = d[1]; k[2] = d[2]; k[3] = d[3]; break; }
        slot = (slot + 1) & (to.cap - 1);
    }
}
cudaError_t launch_set_rehash(SetTable from, SetTable to, cudaStream_t st) {
    k_set_rehash<<<(unsigned)((from.cap + 255) / 256), 256, 0, st>>>(from, to);
    return cudaGetLastError();
}

// multi-GPU merge (pbsgpu_set_allgather): the all-gather delivers [rank][max_n][32] with only counts[rank] valid rows
// per rank; the set wants the digests dense and in global (rank, index) order.  One thread per 8 bytes.
__global__ void k_set_compact_gather(const uint8_t *padded, const uint64_t *counts, uint32_t nranks, uint64_t max_n, uint8_t *dense) {
    const uint32_t r = blockIdx.y;
    uint64_t first = 0;
    for (uint32_t k = 0; k < r; k++) first += counts[k];
    const uint64_t words = counts[r] * 4;
    const uint64_t *src = (const uint64_t *)(padded + (uint64_t)r * max_n * 32);
    uint64_t *dst = (uint64_t *)(dense + first * 32);
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < words; w += (uint64_t)gridDim.x * blockDim.x) dst[w] = src[w];
}
cudaError_t launch_set_compact_gather(const uint8_t *padded, const uint64_t *counts_dev, uint32_t nranks, uint64_t max_n,
                                      uint8_t *dense, cudaStream_t st) {
    if (!nranks || !max_n) return cudaSuccess;
    unsigned bx = (unsigned)std::min<uint64_t>(1024, (max_n * 4 + 255) / 256);
    k_set_compact_gather<<<dim3(bx, nranks), 256, 0, st>>>(padded, counts_dev, nranks, max_n, dense);
    return cudaGetLastError();
}

}  // namespace pbsgpu
