// f3: the hash-chain match search and lazy parse of _lzc DataBlobs (K16, sm_90a).
//
// _lzc is _lzh with another parse: the match of a position is the longest of the first CH_DEPTH entries of its chain
// (every earlier position of the chunk with the same CH_MINMATCH bytes), anywhere up to CH_MAXDIST back in the chunk,
// and the parse is lazy.  tests/zstd_chain_ref.py states every rule; K16 writes K9a's outputs, so K9b and K10 encode the
// blocks unchanged (capi_blob.cu, zstd_frames).  Per pass of whole chunks (CH_PASS_BYTES, or one longer chunk):
//
//   K16a k_ch_keys: per pass position, the key chunk in the pass << 32 | its 4 bytes (LE), or the chunk count << 32
//                  where fewer than 4 bytes are left; the value is the position.
//   sort           cub radix sort (stable) over the key's used bits: equal keys lie side by side in position order.
//   k_ch_prev      prev[v] of every sorted entry: its predecessor's position when that has the same key.
//   K16b k_ch_best: one thread per position of the pass's blocks that are not constant: the chain walk, each candidate
//                  extended byte by byte up to CH_CAP.  best[] = length | offset << 8; 0: no match; CH_SAT: a candidate
//                  reached CH_CAP before the end of the block, so the longest is not known yet.  A long repeat thus
//                  costs CH_CAP bytes per position, not its length.
//   K16c k_ch_parse: one warp per block, all lanes in step (K9a's parser): a ballot over 32 entries of best[] finds the
//                  next match, the literals before it go to the slot one byte per lane, and the lazy steps read the
//                  next entries.  A CH_SAT entry the parse reaches is searched again by the warp, 32 bytes per ballot
//                  step over the full chain walk; the parse jumps past the match, so that costs about
//                  CH_DEPTH * (1 + CH_LAZY) / 32 steps per byte of a long match.
//
// K16d, the DEFLATE instantiation of the same kernels (pbsgpu_deflate_batch_lzc, tests/deflate_chain_ref.py): each
// 128 KiB Deflate segment is one chunk of one block; the key is DCH_MINMATCH bytes, offsets reach DEFLATE_WINDOW, a
// match and K16c's re-search stop at DEFLATE_MAX_MATCH, the gain counts the distance code's extra bits, and a segment
// takes at most LZ_MAX_SEQ matches (the rest are literals).  K15 codes the output unchanged.
#include "internal.cuh"

#include <cub/device/device_radix_sort.cuh>

namespace pbsgpu {

constexpr uint32_t CH_NONE = ~0u;
constexpr uint32_t CH_SAT = 0xFF;          // best[] entry whose longest match K16c finds
constexpr int CH_THREADS = 256;
constexpr uint32_t CH_BEST_SPAN = 8192;    // K16b positions per CTA
static_assert(CH_CAP < CH_SAT, "best[] keeps a length below CH_CAP in 8 bits");

template <bool DEFLATE> struct ChainRule;
template <> struct ChainRule<false> {   // _lzc
    static constexpr uint32_t MINMATCH = CH_MINMATCH, DEPTH = CH_DEPTH, LAZY = CH_LAZY, MAXDIST = CH_MAXDIST;
    static constexpr int MARGIN = CH_MARGIN;
};
template <> struct ChainRule<true> {    // Deflate
    static constexpr uint32_t MINMATCH = DCH_MINMATCH, DEPTH = DCH_DEPTH, LAZY = DCH_LAZY, MAXDIST = DEFLATE_WINDOW;
    static constexpr int MARGIN = DCH_MARGIN;
};
static_assert(DCH_MINMATCH >= 3 && DCH_MINMATCH <= 4 && DEFLATE_MAX_MATCH > CH_CAP, "Deflate keys and lengths");

template <bool DEFLATE>
__global__ void __launch_bounds__(CH_THREADS) k_ch_keys(const ChainArgs a, uint64_t *key, uint32_t *val) {
    using C = ChainRule<DEFLATE>;
    const uint64_t p = (uint64_t)blockIdx.x * CH_THREADS + threadIdx.x;
    if (p >= a.n) return;
    uint32_t lo = a.c0, hi = a.c1 - 1;   // the chunk: the last c with vfirst[c] - vbase <= p
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (a.vfirst[mid] - a.vbase <= p) lo = mid; else hi = mid - 1;
    }
    const uint64_t x = p - (a.vfirst[lo] - a.vbase);
    uint64_t k = (uint64_t)(a.c1 - a.c0) << 32;
    if (x + C::MINMATCH <= a.len[lo]) {
        const uint8_t *q = a.base + a.off[lo] + x;
        k = (uint64_t)(lo - a.c0) << 32 | __ldg(q) | (uint32_t)__ldg(q + 1) << 8 | (uint32_t)__ldg(q + 2) << 16;
        if (C::MINMATCH == 4) k |= (uint32_t)__ldg(q + 3) << 24;
    }
    key[p] = k;
    val[p] = (uint32_t)p;
}

__global__ void __launch_bounds__(CH_THREADS) k_ch_prev(const uint64_t *key, const uint32_t *val, uint64_t n, uint32_t nc,
                                                        uint32_t *prev) {
    const uint64_t k = (uint64_t)blockIdx.x * CH_THREADS + threadIdx.x;
    if (k >= n) return;
    const uint64_t v = key[k];
    prev[val[k]] = k > 0 && key[k - 1] == v && (v >> 32) != nc ? val[k - 1] : CH_NONE;
}

template <bool DEFLATE>
__global__ void __launch_bounds__(CH_THREADS) k_ch_best(const ChainArgs a, const uint32_t *prev, uint32_t *best) {
    using C = ChainRule<DEFLATE>;
    const uint64_t z = a.z0 + blockIdx.x;
    const uint32_t S = a.zsize[z], P = (uint32_t)(a.vpos[z] - a.vbase);
    const uint8_t *p = a.base + a.zsrc[z];
    const uint32_t t1 = min(S, (blockIdx.y + 1) * CH_BEST_SPAN);
    for (uint32_t t = blockIdx.y * CH_BEST_SPAN + threadIdx.x; t < t1; t += CH_THREADS) {
        const uint32_t lim = DEFLATE ? min(S - t, DEFLATE_MAX_MATCH) : S - t, i = P + t;
        uint32_t out = 0;
        if (lim >= C::MINMATCH) {
            const uint32_t cap = min(lim, CH_CAP);
            const uint8_t *q = p + t;
            uint32_t j = prev[i], bl = 0, bo = 0;
            for (uint32_t k = 0; k < C::DEPTH && j != CH_NONE && i - j <= C::MAXDIST; k++) {
                const uint8_t *s = q - (i - j);
                uint32_t L = C::MINMATCH;   // the key's bytes are equal
                while (L < cap && __ldg(s + L) == __ldg(q + L)) L++;
                if (L == cap && cap < lim) { bl = CH_SAT; break; }
                if (L > bl) {
                    bl = L; bo = i - j;
                    if (L == lim) break;
                }
                j = prev[j];
            }
            out = bl == CH_SAT ? CH_SAT : bl | bo << 8;
        }
        best[i] = out;
    }
}

// gain of a match: 4 L - floor(log2(offset + 3)); Deflate: 4 L - the extra bits of the distance code
template <bool DEFLATE> __device__ __forceinline__ int ch_gain(uint32_t L, uint32_t o) {
    if (DEFLATE) return 4 * (int)L - (o <= 2 ? 0 : 30 - __clz(o - 1));
    return 4 * (int)L - (31 - __clz(o + 3));
}

template <bool DEFLATE>
__global__ void __launch_bounds__(128) k_ch_parse(const ChainArgs a, const uint32_t *prev, const uint32_t *best,
                                                  uint64_t first, uint32_t nb, uint8_t *slots, uint64_t *seqs, uint32_t *nseq,
                                                  uint32_t *nlit) {
    const uint32_t w = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    using C = ChainRule<DEFLATE>;
    if (w >= nb) return;
    const uint64_t z = first + w, zo = DEFLATE ? w : z;   // zo: the block's slot and counts
    const uint32_t S = a.zsize[z], P = (uint32_t)(a.vpos[z] - a.vbase);
    const uint8_t *p = a.base + a.zsrc[z];
    const uint32_t *bst = best + P;
    uint8_t *lit = slots + zo * LZ_SLOT + 3;
    uint64_t *sq = seqs + (uint64_t)w * LZ_MAX_SEQ;
    // the match at block position m: best[]'s, or the full chain walk for a CH_SAT entry
    auto match = [&](uint32_t m, uint32_t &L, uint32_t &o) {
        const uint32_t e = bst[m];
        if ((e & 0xFF) != CH_SAT) { L = e & 0xFF; o = e >> 8; return; }
        const uint32_t i = P + m, lim = DEFLATE ? min(S - m, DEFLATE_MAX_MATCH) : S - m;
        const uint8_t *q = p + m;
        uint32_t j = prev[i], bl = 0, bo = 0;
        for (uint32_t k = 0; k < C::DEPTH && j != CH_NONE && i - j <= C::MAXDIST; k++) {
            const uint8_t *s = q - (i - j);
            uint32_t len = 0;
            for (;;) {
                const uint32_t x = len + lane;
                const uint32_t diff = __ballot_sync(~0u, x >= lim || __ldg(s + x) != __ldg(q + x));
                if (diff) { len += __ffs(diff) - 1; break; }
                len += 32;
            }
            if (len > bl) {
                bl = len; bo = i - j;
                if (len == lim) break;
            }
            j = prev[j];
        }
        L = bl; o = bo;
    };
    uint32_t pos = 0, run = 0, nl = 0, ns = 0;   // the same in every lane
    while (pos < S) {
        const uint32_t q = pos + lane;
        const uint32_t hits = __ballot_sync(~0u, (!DEFLATE || ns < LZ_MAX_SEQ) && q < S && bst[q] != 0);
        uint32_t m = hits ? pos + __ffs(hits) - 1 : min(pos + 32, S);
        if (q < m) lit[nl + lane] = __ldg(p + q);
        nl += m - pos;
        pos = m;
        if (!hits) continue;
        uint32_t L, o;
        match(m, L, o);
        for (uint32_t k = 0; k < C::LAZY && m + 1 < S && bst[m + 1] != 0; k++) {
            uint32_t L2, o2;
            match(m + 1, L2, o2);
            if (ch_gain<DEFLATE>(L2, o2) <= ch_gain<DEFLATE>(L, o) + C::MARGIN) break;
            if (lane == 0) lit[nl] = __ldg(p + m);
            nl++; m++; L = L2; o = o2;
        }
        if (lane == 0) sq[ns] = (uint64_t)(m - run) | (uint64_t)L << 20 | (uint64_t)o << 40;
        ns++;
        pos = run = m + L;
    }
    if (lane == 0) { nseq[zo] = ns; nlit[zo] = nl; }
}

// scratch: key[2][n] (u64) | val[2][n] prev[n] (u32) | cub temp; best[] takes the key buffers once prev[] is done
struct ChainLayout { size_t k0, k1, v0, v1, prev, temp, temp_bytes, total; };
static ChainLayout chain_layout(uint64_t n) {
    ChainLayout L;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t tb = 0;
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, tb, k, v, (int)std::max<uint64_t>(n, 1));
    L.k0 = 0; L.k1 = al(n * 8); L.v0 = al(L.k1 + n * 8); L.v1 = al(L.v0 + n * 4); L.prev = al(L.v1 + n * 4);
    L.temp = al(L.prev + n * 4); L.temp_bytes = tb + 256; L.total = L.temp + L.temp_bytes;
    return L;
}
size_t chain_scratch_bytes(uint64_t n) { return chain_layout(n).total; }

#define CH_CK(call) do { const cudaError_t e__ = (call); if (e__ != cudaSuccess) return e__; } while (0)

template <bool DEFLATE> static cudaError_t chain_search(const ChainArgs &a, void *scratch, cudaStream_t st) {
    if (a.z1 <= a.z0 || a.n == 0) return cudaSuccess;
    const ChainLayout L = chain_layout(a.n);
    uint8_t *b = (uint8_t *)scratch;
    uint64_t *k0 = (uint64_t *)(b + L.k0), *k1 = (uint64_t *)(b + L.k1);
    uint32_t *v0 = (uint32_t *)(b + L.v0), *v1 = (uint32_t *)(b + L.v1), *prev = (uint32_t *)(b + L.prev);
    const uint32_t nc = a.c1 - a.c0;
    int end_bit = 32;
    while (end_bit < 64 && (nc >> (end_bit - 32)) != 0) end_bit++;   // the chunk field holds 0 .. nc
    const unsigned g = (unsigned)((a.n + CH_THREADS - 1) / CH_THREADS);
    k_ch_keys<DEFLATE><<<g, CH_THREADS, 0, st>>>(a, k0, v0);
    CH_CK(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> dk(k0, k1);
    cub::DoubleBuffer<uint32_t> dv(v0, v1);
    size_t tb = L.temp_bytes;
    CH_CK(cub::DeviceRadixSort::SortPairs(b + L.temp, tb, dk, dv, (int)a.n, 0, end_bit, st));
    k_ch_prev<<<g, CH_THREADS, 0, st>>>(dk.Current(), dv.Current(), a.n, nc, prev);
    CH_CK(cudaGetLastError());
    const dim3 bg((unsigned)(a.z1 - a.z0), ZFRAME_BLOCK / CH_BEST_SPAN);
    k_ch_best<DEFLATE><<<bg, CH_THREADS, 0, st>>>(a, prev, (uint32_t *)(b + L.k0));
    return cudaGetLastError();
}
static_assert(DEFLATE_SEGMENT == ZFRAME_BLOCK, "K16b's grid covers a Deflate segment as a block");

cudaError_t launch_chain_search(const ChainArgs &a, void *scratch, cudaStream_t st, bool deflate) {
    return deflate ? chain_search<true>(a, scratch, st) : chain_search<false>(a, scratch, st);
}

cudaError_t launch_chain_parse(const ChainArgs &a, const void *scratch, uint64_t first, uint32_t nb, uint8_t *slots,
                               uint64_t *seqs, uint32_t *nseq, uint32_t *nlit, cudaStream_t st, bool deflate) {
    if (nb == 0) return cudaSuccess;
    const ChainLayout L = chain_layout(a.n);
    const uint8_t *b = (const uint8_t *)scratch;
    const uint32_t *prev = (const uint32_t *)(b + L.prev), *best = (const uint32_t *)(b + L.k0);
    if (deflate) k_ch_parse<true><<<(nb + 3) / 4, 128, 0, st>>>(a, prev, best, first, nb, slots, seqs, nseq, nlit);
    else k_ch_parse<false><<<(nb + 3) / 4, 128, 0, st>>>(a, prev, best, first, nb, slots, seqs, nseq, nlit);
    return cudaGetLastError();
}

}  // namespace pbsgpu
