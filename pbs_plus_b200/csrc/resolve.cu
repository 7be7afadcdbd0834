// pbs_plus_b200/csrc/resolve.cu -- K2: sequential min/max rule over sorted candidates.
//
// Replaces ChunkerImpl::shall_break's chunk_size_min / chunk_size_max logic (upstream
// PBS chunker; reached from the reference at internal/pxarmount/commit.go:720 through
// the pxar module).  Closed form: the next cut length is the smallest L in
// [max(min,65), max] with L == max or candidate(start+L-1); the final short chunk is
// emitted at EOF regardless of min.  One thread per stream (the rule is inherently
// sequential per stream; candidates are ~3/2^23 per byte so this is tiny).
#include <cuda_runtime.h>
#include <stdint.h>

#include "internal.cuh"

namespace pbsgpu {

template <bool WRITE>
__global__ void __launch_bounds__(128) k_resolve(ResolveArgs a) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_streams) return;
    unsigned long long nc = *a.cand_count;
    if (nc > a.cand_cap) nc = a.cand_cap;   // overflow is detected and handled by the host (rerun)
    // lower_bound of (s << 40)
    const uint64_t key_lo = (uint64_t)s << KEY_POS_BITS;
    uint64_t lo = 0, hi = nc;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (a.keys_sorted[mid] < key_lo) lo = mid + 1; else hi = mid;
    }
    uint64_t k = lo;
    const uint64_t len = a.len[s];
    const uint64_t min_eff = min_effective(a.cmin);
    uint64_t start = 0;
    uint32_t n = 0;
    uint64_t out = WRITE ? a.chunk_first[s] : 0;
    while (start < len) {
        const uint64_t first_ok = start + min_eff - 1;     // first position scan() may cut after
        uint64_t pos = ~0ull;
        while (k < nc) {
            uint64_t key = a.keys_sorted[k];
            if ((key >> KEY_POS_BITS) != s) break;
            uint64_t p = key & KEY_POS_MASK;
            if (p >= first_ok) { pos = p; break; }
            k++;
        }
        uint64_t end = start + a.cmax;
        if (pos != ~0ull && pos + 1 <= end) end = pos + 1;
        else if (end > len) {
            if (!a.eof) break;         // undecided: needs more data (streaming form)
            end = len;
        }
        if (WRITE && out < a.chunk_cap) {
            ChunkRef c;
            c.stream = s; c.len = (uint32_t)(end - start); c.start = start;
            a.chunks[out] = c;
        }
        out++; n++;
        start = end;
    }
    if (WRITE) { if (a.consumed) a.consumed[s] = start; }
    else a.counts[s] = n;
}

// exclusive scan of counts[n] -> chunk_first[n+1]; single CTA (n is the number of
// streams; 1M streams take ~50 us).
__global__ void __launch_bounds__(1024) k_scan_counts(const uint32_t *counts, uint32_t n, uint64_t *first,
                                                      unsigned long long *total) {
    __shared__ uint64_t warp_sums[32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t base = 0; base < n; base += 1024) {
        uint32_t i = base + threadIdx.x;
        uint64_t v = i < n ? counts[i] : 0, x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = warp_sums[lane], z = w;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, z, d); if (lane >= d) z += y; }
            warp_sums[lane] = z - w;   // exclusive
        }
        __syncthreads();
        uint64_t excl = carry + warp_sums[warp] + x - v;
        if (i < n) first[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) { first[n] = carry; *total = carry; }
}

// Suggested boundaries (pbsgpu_batch_opts.forced_*): appended to the candidate list as ordinary keys "cut after byte
// B-1 of stream s"; the min/max rule above then treats them exactly like hash candidates, which is upstream's
// PayloadChunker rule for byte-wise arrival (a boundary closer than min to the chunk start is skipped, one within
// [min, max] cuts unless a hash candidate comes first, one beyond max waits for the next chunk).
__global__ void k_append_keys(const uint64_t *keys, uint64_t n, uint64_t *cand, uint64_t cand_cap, unsigned long long *cand_count) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long slot = atomicAdd(cand_count, 1ull);
    if (slot < cand_cap) cand[slot] = keys[i];
}
cudaError_t launch_append_keys(const uint64_t *keys, uint64_t n, uint64_t *cand, uint64_t cand_cap, unsigned long long *cand_count,
                               cudaStream_t st) {
    if (!n) return cudaSuccess;
    k_append_keys<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keys, n, cand, cand_cap, cand_count);
    return cudaGetLastError();
}

// Fixed cuts (pbsgpu_batch_opts.fixed_size, the chunking of .fidx images): chunk k of stream s covers
// [k * cs, min((k + 1) * cs, len[s])), so only a stream's last chunk can be short and a stream of length 0 has none.
// No state crosses a chunk boundary, so these launches replace K1, the sort and K2; the ChunkRefs they write are what
// K2 writes for the same cuts, and the back half reads them unchanged.
__global__ void __launch_bounds__(128) k_fixed_counts(const uint64_t *len, uint32_t n, uint32_t cs_log2, uint32_t *counts) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) counts[s] = (uint32_t)((len[s] + (1ull << cs_log2) - 1) >> cs_log2);
}

// One thread per chunk, in (stream, offset) order: the stream is the last s with chunk_first[s] <= t.
__global__ void __launch_bounds__(256) k_fixed_refs(const uint64_t *len, const uint64_t *chunk_first, uint32_t n,
                                                    uint32_t cs_log2, uint64_t n_chunks, ChunkRef *chunks) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_chunks) return;
    uint32_t lo = 0, hi = n;   // upper_bound over chunk_first[1..n]
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (chunk_first[mid + 1] <= t) lo = mid + 1; else hi = mid;
    }
    const uint64_t start = (t - chunk_first[lo]) << cs_log2, l = len[lo] - start;
    ChunkRef c;
    c.stream = lo; c.start = start;
    c.len = (uint32_t)(l < (1ull << cs_log2) ? l : (1ull << cs_log2));
    chunks[t] = c;
}

cudaError_t launch_fixed_refs(const uint64_t *len, uint32_t n, uint32_t cs_log2, uint32_t *counts, uint64_t *chunk_first,
                              unsigned long long *n_chunks_dev, uint64_t n_chunks, ChunkRef *chunks, cudaStream_t st) {
    if (n == 0) return cudaMemsetAsync(n_chunks_dev, 0, sizeof(unsigned long long), st);
    k_fixed_counts<<<(n + 127) / 128, 128, 0, st>>>(len, n, cs_log2, counts);
    k_scan_counts<<<1, 1024, 0, st>>>(counts, n, chunk_first, n_chunks_dev);
    if (n_chunks) k_fixed_refs<<<(unsigned)((n_chunks + 255) / 256), 256, 0, st>>>(len, chunk_first, n, cs_log2, n_chunks, chunks);
    return cudaGetLastError();
}

cudaError_t launch_resolve(const ResolveArgs &a, cudaStream_t st) {
    if (a.n_streams == 0) return cudaMemsetAsync(a.n_chunks, 0, sizeof(unsigned long long), st);
    unsigned blocks = (a.n_streams + 127) / 128;
    k_resolve<false><<<blocks, 128, 0, st>>>(a);
    k_scan_counts<<<1, 1024, 0, st>>>(a.counts, a.n_streams, a.chunk_first, a.n_chunks);
    k_resolve<true><<<blocks, 128, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace pbsgpu
