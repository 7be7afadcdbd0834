// f3: long-distance matches of _lzl DataBlobs (K12, sm_90a).
//
// _lzl is _lzh plus long matches that reach anywhere earlier in the same chunk.  K12 finds them per pass of whole chunks
// (LDM_PASS_BYTES; tests/zstd_ldm_ref.py states every rule below); the host splits the kept ones at the 128 KiB block
// edges into long spans, and K9a's span parse, K9b and K10 encode the blocks that hold one (capi_blob.cu, zstd_frames).
//
//   anchor    position i >= 63 of a chunk whose gear hash h = sum_k G[byte i-k] << k (k < 64) has its top LDM_RATE bits
//             zero; the fingerprint is h.  G is splitmix64 from LDM_SEED.
//   cand(a)   the latest earlier anchor of the chunk with a's fingerprint, at most LDM_MAXDIST back, whose window equals
//             a's.  Its match [s, e) at offset d = a - cand(a) is the window extended while the bytes at x and x - d
//             are equal, backward down to s = d (the source stays in the chunk) and forward to the chunk end.
//   selection by (s, e descending, d): cur = 0, s' = max(s, cur); [s', e) is kept when e - s' >= LDM_MINMATCH, cur = e.
//
//   K12a k_ldm_scan<false>: one thread per LDM_SPAN positions (63 bytes of warm-up, G in shared memory) counts its anchors;
//                  cub's exclusive sum places them, and k_ldm_scan<true> writes (fingerprint, chunk << 40 | position in
//                  the pass) in position order.
//   sort 1         cub radix sort by fingerprint (stable): cand(a) is a's predecessor when it has the same key and chunk.
//   K12b k_ldm_cand: per anchor with a predecessor in reach, the key offset << 40 | position; none = all ones.
//   sort 2         by (offset, position): the candidates of one diagonal of a chunk lie side by side in position order.
//   K12c k_ldm_extend: one warp per candidate, 32 bytes per ballot step.  The window is compared; a candidate whose
//                  diagonal neighbour before it is a valid window joined to it by equal bytes lies in that neighbour's
//                  run and gives the same match, so only the first candidate of each run extends (a long copy costs
//                  its length once, not once per anchor).  Out: chunk << 40 | s, offset << 40 | e.
//   sort 3         by (chunk, s).
//   K12d k_ldm_select: one thread per chunk walks its matches in that order: among the matches with one s the longest
//                  (then the nearest) is the only one that can be kept, so it alone is tested against cur.  Kept
//                  matches are appended (atomic count) and go to the host, which sorts and splits them.
#include "internal.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace pbsgpu {

constexpr int LDM_THREADS = 256;
constexpr uint64_t NONE = ~0ull;

__device__ __forceinline__ uint64_t ldm_gear(uint32_t k) {   // splitmix64's k-th output
    uint64_t z = LDM_SEED + (uint64_t)(k + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// WRITE = false: per span its anchor count (cnt, may be NULL) and the pass total (total, may be NULL);
// WRITE = true: the anchors of span t at at[t - s0] ..
template <bool WRITE>
__global__ void __launch_bounds__(LDM_THREADS) k_ldm_scan(const LdmArgs a, uint64_t *cnt, unsigned long long *total,
                                                          const uint64_t *at, uint64_t *fp, uint64_t *val) {
    __shared__ uint64_t G[256];
    G[threadIdx.x] = ldm_gear(threadIdx.x);
    __syncthreads();
    const uint64_t t = a.s0 + (uint64_t)blockIdx.x * LDM_THREADS + threadIdx.x;
    uint32_t n = 0;
    if (t < a.s1) {
        uint32_t lo = a.c0, hi = a.c1 - 1;   // the chunk: the last i with span_first[i] <= t
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) / 2;
            if (a.span_first[mid] <= t) lo = mid; else hi = mid - 1;
        }
        const uint8_t *p = a.base + a.off[lo];
        const uint64_t p0 = LDM_WINDOW - 1 + (t - a.span_first[lo]) * LDM_SPAN, p1 = min(p0 + LDM_SPAN, a.len[lo]);
        const uint64_t v = (uint64_t)(lo - a.c0) << 40 | (a.vfirst[lo] - a.vfirst[a.c0]);
        uint64_t h = 0, w = WRITE ? at[t - a.s0] : 0;
        for (uint64_t x = p0 - (LDM_WINDOW - 1); x < p1; x++) {
            h = (h << 1) + G[__ldg(p + x)];
            if (x >= p0 && (h >> (64 - LDM_RATE)) == 0) {
                if (WRITE) { fp[w] = h; val[w] = v + x; w++; }
                else n++;
            }
        }
        if (!WRITE && cnt) cnt[t - a.s0] = n;
    }
    if (!WRITE && total) {
        n = __reduce_add_sync(~0u, n);
        if ((threadIdx.x & 31) == 0 && n) atomicAdd(total, (unsigned long long)n);
    }
}

__global__ void k_ldm_cand(const uint64_t *fp, const uint64_t *val, uint64_t n, uint64_t *key, uint64_t *chunk) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t v = val[i];
    uint64_t k = NONE;
    if (i > 0 && fp[i - 1] == fp[i] && (val[i - 1] >> 40) == (v >> 40) && v - val[i - 1] <= LDM_MAXDIST)
        k = (v - val[i - 1]) << 40 | (v & LDM_M40);
    key[i] = k;
    chunk[i] = v >> 40;
}

// the 64-byte windows ending at x and x - d are equal (two bytes per lane)
__device__ __forceinline__ bool window_eq(const uint8_t *p, uint64_t x, uint64_t d, uint32_t lane) {
    const uint64_t y = x - (LDM_WINDOW - 1) + lane, z = y + 32;
    return __all_sync(~0u, __ldg(p + y) == __ldg(p + y - d) && __ldg(p + z) == __ldg(p + z - d));
}

// the bytes at y and y - d are equal for every y in [lo, hi)
__device__ __forceinline__ bool run_eq(const uint8_t *p, uint64_t lo, uint64_t hi, uint64_t d, uint32_t lane) {
    for (uint64_t y = lo; y < hi; y += 32) {
        const uint64_t q = y + lane;
        if (__any_sync(~0u, q < hi && __ldg(p + q) != __ldg(p + q - d))) return false;
    }
    return true;
}

__global__ void __launch_bounds__(LDM_THREADS) k_ldm_extend(const LdmArgs a, const uint64_t *ckey, const uint64_t *cchunk,
                                                            uint64_t n, uint64_t *mkey, uint64_t *mval) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t i = ((uint64_t)blockIdx.x * LDM_THREADS + threadIdx.x) >> 5;
    if (i >= n) return;
    const uint64_t k = ckey[i];
    uint64_t ok = NONE, ov = 0;
    if (k != NONE) {
        const uint64_t d = k >> 40, cl = cchunk[i];
        const uint32_t c = a.c0 + (uint32_t)cl;
        const uint8_t *p = a.base + a.off[c];
        const uint64_t len = a.len[c], vb = a.vfirst[c] - a.vfirst[a.c0], x = (k & LDM_M40) - vb;
        bool lead = window_eq(p, x, d, lane);
        if (lead && i > 0 && ckey[i - 1] != NONE && (ckey[i - 1] >> 40) == d && cchunk[i - 1] == cl) {
            const uint64_t xp = (ckey[i - 1] & LDM_M40) - vb;
            lead = !(window_eq(p, xp, d, lane) && run_eq(p, xp + 1, x - (LDM_WINDOW - 1), d, lane));
        }
        if (lead) {
            uint64_t s = x - (LDM_WINDOW - 1), e = x + 1;
            for (;;) {   // lane l looks at s - 1 - l; the run stops below d or at a difference
                const uint64_t y = s - 1 - lane;
                const uint32_t stop = __ballot_sync(~0u, s - d <= lane || __ldg(p + y) != __ldg(p + y - d));
                if (stop) { s -= __ffs(stop) - 1; break; }
                s -= 32;
            }
            for (;;) {
                const uint64_t y = e + lane;
                const uint32_t stop = __ballot_sync(~0u, y >= len || __ldg(p + y) != __ldg(p + y - d));
                if (stop) { e += __ffs(stop) - 1; break; }
                e += 32;
            }
            ok = cl << 40 | s;
            ov = d << 40 | e;
        }
    }
    if (lane == 0) { mkey[i] = ok; mval[i] = ov; }
}

__global__ void k_ldm_select(const uint64_t *mkey, const uint64_t *mval, uint64_t n, uint32_t nc, uint64_t *kkey,
                             uint64_t *kval, uint32_t *n_kept) {
    const uint32_t cl = blockIdx.x * blockDim.x + threadIdx.x;
    if (cl >= nc) return;
    uint64_t lo = 0, hi = n;   // the first match of chunk cl
    while (lo < hi) {
        const uint64_t mid = (lo + hi) / 2;
        if ((mkey[mid] >> 40) < cl) lo = mid + 1; else hi = mid;
    }
    uint64_t cur = 0;
    for (uint64_t j = lo; j < n && (mkey[j] >> 40) == cl;) {
        const uint64_t k = mkey[j], s = k & LDM_M40;
        uint64_t e = mval[j] & LDM_M40, d = mval[j] >> 40;
        for (j++; j < n && mkey[j] == k; j++) {
            const uint64_t e2 = mval[j] & LDM_M40, d2 = mval[j] >> 40;
            if (e2 > e || (e2 == e && d2 < d)) { e = e2; d = d2; }
        }
        const uint64_t s2 = max(s, cur);
        if (e >= s2 + LDM_MINMATCH) {
            const uint32_t w = atomicAdd(n_kept, 1u);
            kkey[w] = (uint64_t)cl << 40 | s2;
            kval[w] = d << 40 | e;
            cur = e;
        }
    }
}

cudaError_t launch_ldm_count(const LdmArgs &a, unsigned long long *total, cudaStream_t st) {
    if (a.s1 <= a.s0) return cudaSuccess;
    k_ldm_scan<false><<<(unsigned)((a.s1 - a.s0 + LDM_THREADS - 1) / LDM_THREADS), LDM_THREADS, 0, st>>>(a, nullptr, total, nullptr,
                                                                                                     nullptr, nullptr);
    return cudaGetLastError();
}

// scratch: cnt[spans] at[spans] (u64) | k0 k1 v0 v1 [anchors] (u64) | n_kept | cub temp
struct LdmLayout { size_t cnt, at, k0, k1, v0, v1, nk, temp, temp_bytes, total; };
static LdmLayout ldm_layout(uint64_t spans, uint64_t anchors) {
    LdmLayout L;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t ts = 0, tr = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, ts, (uint64_t *)nullptr, (uint64_t *)nullptr, (int)std::max<uint64_t>(spans, 1));
    cub::DeviceRadixSort::SortPairs(nullptr, tr, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                    (int)std::max<uint64_t>(anchors, 1));
    L.cnt = 0; L.at = al(spans * 8); L.k0 = al(L.at + spans * 8); L.k1 = al(L.k0 + anchors * 8);
    L.v0 = al(L.k1 + anchors * 8); L.v1 = al(L.v0 + anchors * 8); L.nk = al(L.v1 + anchors * 8); L.temp = al(L.nk + 4);
    L.temp_bytes = std::max(ts, tr) + 256; L.total = L.temp + L.temp_bytes;
    return L;
}
size_t ldm_scratch_bytes(uint64_t spans, uint64_t anchors) { return ldm_layout(spans, anchors).total; }

#define LDM_CK(call) do { const cudaError_t e__ = (call); if (e__ != cudaSuccess) return e__; } while (0)

cudaError_t launch_ldm_matches(const LdmArgs &a, uint64_t anchors, void *scratch, uint64_t **key, uint64_t **val,
                               uint32_t **n_kept, cudaStream_t st) {
    const uint64_t ns = a.s1 - a.s0;
    const LdmLayout L = ldm_layout(ns, anchors);
    uint8_t *b = (uint8_t *)scratch;
    uint64_t *cnt = (uint64_t *)(b + L.cnt), *at = (uint64_t *)(b + L.at), *k0 = (uint64_t *)(b + L.k0);
    uint64_t *k1 = (uint64_t *)(b + L.k1), *v0 = (uint64_t *)(b + L.v0), *v1 = (uint64_t *)(b + L.v1);
    uint32_t *nk = (uint32_t *)(b + L.nk);
    *key = k0; *val = v0; *n_kept = nk;
    LDM_CK(cudaMemsetAsync(nk, 0, 4, st));
    if (anchors < 2) return cudaSuccess;
    size_t tb = L.temp_bytes;
    const unsigned sg = (unsigned)((ns + LDM_THREADS - 1) / LDM_THREADS);
    k_ldm_scan<false><<<sg, LDM_THREADS, 0, st>>>(a, cnt, nullptr, nullptr, nullptr, nullptr);
    LDM_CK(cudaGetLastError());
    LDM_CK(cub::DeviceScan::ExclusiveSum(b + L.temp, tb, cnt, at, (int)ns, st));
    k_ldm_scan<true><<<sg, LDM_THREADS, 0, st>>>(a, nullptr, nullptr, at, k0, v0);
    LDM_CK(cudaGetLastError());
    tb = L.temp_bytes;
    LDM_CK(cub::DeviceRadixSort::SortPairs(b + L.temp, tb, k0, k1, v0, v1, (int)anchors, 0, 64 - LDM_RATE, st));
    const unsigned ag = (unsigned)((anchors + LDM_THREADS - 1) / LDM_THREADS);
    k_ldm_cand<<<ag, LDM_THREADS, 0, st>>>(k1, v1, anchors, k0, v0);
    LDM_CK(cudaGetLastError());
    tb = L.temp_bytes;
    LDM_CK(cub::DeviceRadixSort::SortPairs(b + L.temp, tb, k0, k1, v0, v1, (int)anchors, 0, 64, st));
    k_ldm_extend<<<(unsigned)((anchors * 32 + LDM_THREADS - 1) / LDM_THREADS), LDM_THREADS, 0, st>>>(a, k1, v1, anchors, k0, v0);
    LDM_CK(cudaGetLastError());
    tb = L.temp_bytes;
    LDM_CK(cub::DeviceRadixSort::SortPairs(b + L.temp, tb, k0, k1, v0, v1, (int)anchors, 0, 64, st));
    const uint32_t nc = a.c1 - a.c0;
    k_ldm_select<<<(nc + 127) / 128, 128, 0, st>>>(k1, v1, anchors, nc, k0, v0, nk);
    return cudaGetLastError();
}

}  // namespace pbsgpu
