// f3, read side: raw Deflate streams (RFC 1951) of restored files, the zip restore's compression (K15, sm_90a).
//
// A range is cut into DEFLATE_SEGMENT-byte segments that are coded independently: K9a's greedy parse with the Deflate
// limits (zlz.cu, k_lz_parse<false, true>), then K15 writes each segment as the smallest of three forms -- stored
// blocks, one fixed-code block, one dynamic-code block -- stored then fixed on ties.  A form's cost counts the
// segment's end (BFINAL and padding on the stream's last segment, else an empty stored block behind a fixed or dynamic
// block), so every segment ends byte-aligned and is never larger than its stored form.  tests/deflate_ref.py states the
// format and each rule below.
//
//   K15 k_deflate_encode: one CTA of 256 threads per segment.
//     1. every thread takes a run of sequences: lit/len and distance histograms in shared memory, a CTA scan of the
//        literal lengths rewrites each packed sequence's literal length as the end of its literals (litend_k); the
//        literal histogram is strided over the literals;
//     2. warp 0 builds the lit/len, distance and code-length codes (huf_lengths, zent.cuh), the run-length coded code
//        lengths and the bit counts of the three forms;
//     3. stored: the CTA copies the blocks.  Otherwise each thread takes a run of the token stream (literals and
//        matches in stream order; match k is token litend_k + k), a CTA scan of its bit cost places it, and it ORs its
//        codes into the zeroed output in 32-bit words, as K10 places its Huffman streams.
#include "internal.cuh"

namespace pbsgpu {

constexpr int DEF_THREADS = 256;
enum : uint32_t { FORM_STORED = 0, FORM_FIXED = 1, FORM_DYNAMIC = 2 };

__constant__ uint16_t DEF_LEN_BASE[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                          31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint16_t DEF_DIST_BASE[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                           193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t DEF_CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// length code - 257 of a match length 3..258, and its extra bits
__device__ __forceinline__ uint32_t len_code(uint32_t L) {
    const uint32_t v = L - 3;
    if (L == 258) return 28;
    if (v < 8) return v;
    const uint32_t lg = 31 - __clz(v);
    return 4 * (lg - 1) + ((v >> (lg - 2)) & 3);
}
__device__ __forceinline__ uint32_t len_bits(uint32_t c) { return c < 8 || c == 28 ? 0 : c / 4 - 1; }
// distance code of a distance 1..32768, and its extra bits
__device__ __forceinline__ uint32_t dist_code(uint32_t d) {
    if (d <= 2) return d - 1;
    const uint32_t lg = 31 - __clz(d - 1);
    return 2 * lg + (((d - 1) >> (lg - 1)) & 1);
}
__device__ __forceinline__ uint32_t dist_bits(uint32_t c) { return c < 4 ? 0 : c / 2 - 1; }

struct DefShared {
    uint32_t lhist[288], dhist[32], clhist[19];
    // huf_lengths scratch, sized for the lit/len alphabet
    uint32_t hc[288], hw[2 * 286];
    uint16_t hparent[2 * 286], horder[286];
    uint8_t hdepth[2 * 286];
    uint8_t llen[288], dlen[32], cllen[19];
    uint16_t lcode[288], dcode[32], clcode[19];   // bit-reversed canonical codes
    uint8_t rsym[286 + 30], rval[286 + 30];       // the run-length coded code lengths
    uint32_t wsum[DEF_THREADS / 32], next[16];
    uint32_t nruns, hlit, hdist, hclen, hdr_bits, form, bytes, maxlen;
};

// exclusive prefix sum over the CTA; *total = the sum of all
__device__ uint32_t cta_scan(uint32_t v, uint32_t *wsum, uint32_t *total) {
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(~0u, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (uint32_t k = 0; k < DEF_THREADS / 32; k++) { before += k < w ? wsum[k] : 0; all += wsum[k]; }
    __syncthreads();   // wsum is reused by the next scan
    *total = all;
    return before + x - v;
}

__device__ __forceinline__ uint32_t rev(uint32_t code, uint32_t len) { return __brev(code) >> (32 - len); }

// canonical codes (RFC 1951 3.2.2) of lengths len[0..n), bit-reversed for the LSB-first writer (one thread); next[16]
// is shared scratch
__device__ void def_canonical(const uint8_t *len, uint32_t n, uint16_t *code, uint32_t *next) {
    for (uint32_t b = 0; b < 16; b++) next[b] = 0;
    for (uint32_t x = 0; x < n; x++) next[len[x]]++;
    for (uint32_t b = 1, c = 0, prev = 0; b < 16; b++) { c = (c + prev) << 1; prev = next[b]; next[b] = c; }
    for (uint32_t x = 0; x < n; x++) if (len[x]) code[x] = (uint16_t)rev(next[len[x]]++, len[x]);
}

// code lengths of cnt[0..n) at most `limit` bits into len[] (warp 0): one present symbol gets length 1
__device__ void def_lengths(DefShared &s, const uint32_t *cnt, uint32_t n, uint32_t limit, uint8_t *len, uint32_t lane) {
    uint32_t m = 0, one = 0;
    for (uint32_t x = lane; x < n; x += 32) if (cnt[x]) { m++; one = x; }
    m = __reduce_add_sync(~0u, m);
    one = __reduce_max_sync(~0u, one);
    for (uint32_t x = lane; x < n; x += 32) len[x] = 0;
    __syncwarp();
    if (m == 1 && lane == 0) len[one] = 1;
    if (m >= 2) huf_lengths(cnt, n, m, limit, lane, s.hc, s.horder, s.hw, s.hparent, s.hdepth, len, &s.maxlen);
    __syncwarp();
}

// Appends bits LSB first to 32-bit words by atomicOr (neighbouring threads share words); the words are zeroed.
struct OrBits {
    uint32_t *w;
    uint32_t at, na = 0;
    uint64_t acc = 0;
    __device__ OrBits(uint32_t *words, uint32_t bit) : w(words + (bit >> 5)), at(0), na(bit & 31) {}
    __device__ void add(uint32_t v, uint32_t nb) {
        acc |= (uint64_t)v << na;
        na += nb;
        if (na >= 32) { atomicOr(w + at, (uint32_t)acc); acc >>= 32; na -= 32; at++; }
    }
    __device__ void flush() { if (na) atomicOr(w + at, (uint32_t)acc); }
};

__global__ void __launch_bounds__(DEF_THREADS) k_deflate_encode(const uint8_t *base, const uint64_t *src, const uint32_t *size,
                                                                const uint8_t *final_, const uint8_t *lits, uint64_t *seqs,
                                                                const uint32_t *nseq, const uint32_t *nlit, uint8_t *out,
                                                                uint32_t *out_len) {
    __shared__ DefShared s;
    const uint32_t tid = threadIdx.x, lane = tid & 31, g = blockIdx.x;
    const uint32_t S = size[g], n = nseq[g], nl = nlit[g];
    const bool fin = final_[g] != 0;
    const uint8_t *lit = lits + (uint64_t)g * LZ_SLOT + 3;
    uint64_t *sq = seqs + (uint64_t)g * LZ_MAX_SEQ;
    uint8_t *o = out + (uint64_t)g * DEFLATE_SLOT;

    for (uint32_t k = tid; k < 288; k += DEF_THREADS) s.lhist[k] = 0;
    if (tid < 32) s.dhist[tid] = 0;
    if (tid < 19) s.clhist[tid] = 0;
    __syncthreads();
    // 1. histograms; literal lengths -> litend
    {
        const uint32_t per = (n + DEF_THREADS - 1) / DEF_THREADS, k0 = min(tid * per, n), k1 = min(k0 + per, n);
        uint32_t v = 0, tot;
        for (uint32_t k = k0; k < k1; k++) {
            const uint64_t q = sq[k];
            v += (uint32_t)(q & 0xFFFFF);
            atomicAdd(&s.lhist[257 + len_code((uint32_t)(q >> 20) & 0xFFFFF)], 1u);
            atomicAdd(&s.dhist[dist_code((uint32_t)(q >> 40))], 1u);
        }
        uint32_t e = cta_scan(v, s.wsum, &tot);
        for (uint32_t k = k0; k < k1; k++) {
            const uint64_t q = sq[k];
            e += (uint32_t)(q & 0xFFFFF);
            sq[k] = (q & ~0xFFFFFull) | e;
        }
        for (uint32_t i = tid; i < nl; i += DEF_THREADS) atomicAdd(&s.lhist[lit[i]], 1u);
        if (tid == 0) s.lhist[256] = 1;   // end of block
    }
    __syncthreads();
    // 2. the codes and the form (warp 0)
    const uint32_t nst = (S + DEFLATE_STORED_MAX - 1) / DEFLATE_STORED_MAX;
    if (tid < 32) {
        def_lengths(s, s.lhist, 286, DEFLATE_MAXBITS, s.llen, lane);
        def_lengths(s, s.dhist, 30, DEFLATE_MAXBITS, s.dlen, lane);
        uint32_t hl = 0, hd = 0;
        for (uint32_t x = lane; x < 286; x += 32) if (s.llen[x]) hl = x + 1;
        for (uint32_t x = lane; x < 30; x += 32) if (s.dlen[x]) hd = x + 1;
        hl = max(257u, __reduce_max_sync(~0u, hl));
        hd = __reduce_max_sync(~0u, hd);
        if (lane == 0) {
            if (hd == 0) { s.dlen[0] = 1; hd = 1; }   // no matches: one distance code of length 1
            s.hlit = hl; s.hdist = hd;
            // greedy run-length coding of lit/len lengths [0, hlit) then distance lengths [0, hdist)
            const uint32_t tot = hl + hd;
            auto L = [&](uint32_t i) -> uint32_t { return i < hl ? s.llen[i] : s.dlen[i - hl]; };
            uint32_t nr = 0;
            for (uint32_t i = 0; i < tot;) {
                const uint32_t v = L(i);
                uint32_t r = 1;
                while (i + r < tot && L(i + r) == v) r++;
                if (v == 0 && r >= 11) { const uint32_t k = min(r, 138u); s.rsym[nr] = 18; s.rval[nr++] = k - 11; i += k; }
                else if (v == 0 && r >= 3) { s.rsym[nr] = 17; s.rval[nr++] = r - 3; i += r; }
                else {
                    s.rsym[nr] = v; s.rval[nr++] = 0; i++; r--;
                    while (v && r >= 3) { const uint32_t k = min(r, 6u); s.rsym[nr] = 16; s.rval[nr++] = k - 3; i += k; r -= k; }
                }
            }
            s.nruns = nr;
            for (uint32_t k = 0; k < nr; k++) s.clhist[s.rsym[k]]++;
        }
        __syncwarp();
        def_lengths(s, s.clhist, 19, DEFLATE_CL_MAXBITS, s.cllen, lane);
        // bit counts: the token stream under each code, plus the extra bits both forms share
        uint32_t fx = 0, dy = 0, ex = 0;
        for (uint32_t x = lane; x < 286; x += 32) {
            const uint32_t c = s.lhist[x], fl = x < 144 ? 8 : x < 256 ? 9 : x < 280 ? 7 : 8;
            fx += c * fl; dy += c * s.llen[x];
            if (x >= 257) ex += c * len_bits(x - 257);
        }
        if (lane < 30) { const uint32_t c = s.dhist[lane]; fx += c * 5; dy += c * s.dlen[lane]; ex += c * dist_bits(lane); }
        fx = __reduce_add_sync(~0u, fx); dy = __reduce_add_sync(~0u, dy); ex = __reduce_add_sync(~0u, ex);
        if (lane == 0) {
            uint32_t hclen = 19;
            while (hclen > 4 && s.cllen[DEF_CL_ORDER[hclen - 1]] == 0) hclen--;
            s.hclen = hclen;
            uint32_t hdr = 3 + 14 + 3 * hclen;
            for (uint32_t k = 0; k < s.nruns; k++) {
                const uint32_t y = s.rsym[k];
                hdr += s.cllen[y] + (y == 16 ? 2 : y == 17 ? 3 : y == 18 ? 7 : 0);
            }
            const uint32_t fixed_bits = 3 + fx + ex, dyn_bits = hdr + dy + ex;
            auto total = [&](uint32_t b) { return fin ? (b + 7) / 8 * 8 : (b + 3 + 7) / 8 * 8 + 32; };
            const uint32_t cs = 40 * nst + 8 * S, cf = total(fixed_bits), cd = total(dyn_bits);
            uint32_t form = FORM_STORED, best = cs;
            if (cf < best) { form = FORM_FIXED; best = cf; }
            if (cd < best) { form = FORM_DYNAMIC; best = cd; }
            s.form = form; s.bytes = best / 8;
            s.hdr_bits = form == FORM_FIXED ? 3 : hdr;
            if (form == FORM_FIXED) {   // RFC 1951 3.2.6
                for (uint32_t x = 0; x < 288; x++) s.llen[x] = x < 144 ? 8 : x < 256 ? 9 : x < 280 ? 7 : 8;
                for (uint32_t x = 0; x < 30; x++) s.dlen[x] = 5;
            }
            if (form != FORM_STORED) {
                def_canonical(s.llen, form == FORM_FIXED ? 288 : 286, s.lcode, s.next);
                def_canonical(s.dlen, 30, s.dcode, s.next);
                def_canonical(s.cllen, 19, s.clcode, s.next);
            }
            out_len[g] = best / 8;
        }
    }
    __syncthreads();
    const uint32_t form = s.form, bytes = s.bytes;
    const uint8_t *p = base + src[g];
    if (form == FORM_STORED) {
        for (uint32_t k = 0; k < nst; k++) {
            const uint32_t a = k * DEFLATE_STORED_MAX, len = min(S - a, DEFLATE_STORED_MAX), at = a + 5 * k;
            if (tid == 0) {
                o[at] = fin && k + 1 == nst;
                o[at + 1] = (uint8_t)len; o[at + 2] = (uint8_t)(len >> 8);
                o[at + 3] = (uint8_t)~len; o[at + 4] = (uint8_t)(~len >> 8);
            }
            for (uint32_t i = tid; i < len; i += DEF_THREADS) o[at + 5 + i] = p[a + i];
        }
        return;
    }
    uint32_t *W = (uint32_t *)o;
    for (uint32_t k = tid; k < (bytes + 3) / 4; k += DEF_THREADS) W[k] = 0;
    __syncthreads();
    // 3. the token stream: literal j of sequence k is token j + k, match k is token litend_k + k
    const uint32_t T = nl + n, per = (T + DEF_THREADS - 1) / DEF_THREADS, x0 = min(tid * per, T), x1 = min(x0 + per, T);
    uint32_t k0 = 0;
    {
        uint32_t lo = 0, hi = n;   // the first match k with token index >= x0
        while (lo < hi) {
            const uint32_t mid = (lo + hi) / 2;
            if ((uint32_t)(sq[mid] & 0xFFFFF) + mid < x0) lo = mid + 1; else hi = mid;
        }
        k0 = lo;
    }
    uint32_t cost = 0;
    for (uint32_t x = x0, k = k0; x < x1; x++) {
        if (k < n && x == (uint32_t)(sq[k] & 0xFFFFF) + k) {
            const uint64_t q = sq[k++];
            const uint32_t lc = len_code((uint32_t)(q >> 20) & 0xFFFFF), dc = dist_code((uint32_t)(q >> 40));
            cost += s.llen[257 + lc] + len_bits(lc) + s.dlen[dc] + dist_bits(dc);
        } else {
            cost += s.llen[lit[x - k]];
        }
    }
    uint32_t tot;
    const uint32_t start = s.hdr_bits + cta_scan(cost, s.wsum, &tot);
    if (x0 < x1) {
        OrBits w(W, start);
        for (uint32_t x = x0, k = k0; x < x1; x++) {
            if (k < n && x == (uint32_t)(sq[k] & 0xFFFFF) + k) {
                const uint64_t q = sq[k++];
                const uint32_t L = (uint32_t)(q >> 20) & 0xFFFFF, d = (uint32_t)(q >> 40);
                const uint32_t lc = len_code(L), dc = dist_code(d);
                w.add(s.lcode[257 + lc], s.llen[257 + lc]);
                w.add(L - DEF_LEN_BASE[lc], len_bits(lc));
                w.add(s.dcode[dc], s.dlen[dc]);
                w.add(d - DEF_DIST_BASE[dc], dist_bits(dc));
            } else {
                const uint32_t b = lit[x - k];
                w.add(s.lcode[b], s.llen[b]);
            }
        }
        w.flush();
    }
    if (tid == 0) {   // block header and code description, then end of block and the segment's end
        OrBits w(W, 0);
        w.add(fin, 1);
        if (form == FORM_FIXED) w.add(1, 2);
        else {
            w.add(2, 2);
            w.add(s.hlit - 257, 5); w.add(s.hdist - 1, 5); w.add(s.hclen - 4, 4);
            for (uint32_t k = 0; k < s.hclen; k++) w.add(s.cllen[DEF_CL_ORDER[k]], 3);
            for (uint32_t k = 0; k < s.nruns; k++) {
                const uint32_t y = s.rsym[k];
                w.add(s.clcode[y], s.cllen[y]);
                if (y >= 16) w.add(s.rval[k], y == 16 ? 2 : y == 17 ? 3 : 7);
            }
        }
        w.flush();
        const uint32_t end = s.hdr_bits + tot + s.llen[256];
        OrBits e(W, end - s.llen[256]);
        e.add(s.lcode[256], s.llen[256]);
        if (!fin) {   // an empty non-final stored block: 3 zero bits, padding, LEN 0, NLEN 0xFFFF
            e.add(0, 3 + (8 - (end + 3) % 8) % 8);
            e.add(0, 16); e.add(0xFFFF, 16);
        }
        e.flush();
    }
}

cudaError_t launch_deflate_encode(const uint8_t *base, const uint64_t *src, const uint32_t *size, const uint8_t *final_,
                                  uint32_t nb, const uint8_t *lits, uint64_t *seqs, const uint32_t *nseq,
                                  const uint32_t *nlit, uint8_t *out, uint32_t *out_len, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    k_deflate_encode<<<nb, DEF_THREADS, 0, st>>>(base, src, size, final_, lits, seqs, nseq, nlit, out, out_len);
    return cudaGetLastError();
}

}  // namespace pbsgpu
