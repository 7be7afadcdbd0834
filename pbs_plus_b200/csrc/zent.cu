// f3: zstd's entropy stage for compressed DataBlobs (K10, sm_90a): FSE_Compressed_Mode sequences, Huffman literals.
//
// K10 re-encodes what K9a parsed.  Per block of a pass, after K9b: the literals K9a left at slot + 3 and the sequences
// in the pass scratch are coded with the block's own tables, and that Block_Content replaces K9b's (in the slot and in
// info[g]) when it is smaller than K9b's and than the block.  tests/zstd_ent_ref.py (block_content) states the format;
// each rule below is also stated and commented there.
//
//   sequences  LL, OF, ML columns: RLE_Mode when every sequence has the same code, else FSE_Compressed_Mode with
//              log = min(cap, max(5, bit_length(n) - 2)), raised until 2^log >= the codes present (caps LL 9, OF 8,
//              ML 9), and the distribution normalised as in ent_table.  Offsets stay offset + 3, so no Repeat_Mode;
//              the bitstream is seq_bitstream's, as K9b's, with these tables.
//   literals   RLE_Literals_Block when all have one value; Huffman (Compressed_Literals_Block, direct 4-bit weights) when
//              there are >= 2 values, none above 128, and that section is smaller than the raw one; else raw.  Code
//              lengths <= 11 (two-queue Huffman, counts halved until the longest fits), canonical codes.  One stream
//              when the regenerated and compressed sizes both fit 10 bits, else four behind the jump table.
//   full       (FULL, the _lzh encoder; tests/zstd_huf_ref.py): Huffman literals whatever their largest value, the
//              tree in the smaller allowed form of the direct one and the FSE-compressed weights (ent_fse_tree), the
//              direct one on ties; raw when neither is allowed.  Never larger than the content with FULL off.
//
// One CTA of 256 threads per block: shared-memory histograms (all threads); then warp 0 builds the Huffman code while
// lane 0 of warps 1..3 builds the LL / OF / ML tables; then lane 0 of warp 7 runs the serial FSE chain into the
// scratch while warps 0..6 write the Huffman streams (a scan of the code lengths places every thread's run of literals;
// 32-bit atomicOr into zeroed scratch, since neighbouring runs share words); finally the CTA copies the chosen content
// over the slot.  The content never overwrites the literals it is still reading: it is built in scratch first.
#include "internal.cuh"

namespace pbsgpu {

constexpr int ENT_THREADS = 256;
constexpr int ENT_WRITERS = ENT_THREADS - 32;   // warps 0..6 write the literals; lane 0 of warp 7 runs the FSE chain
enum : uint32_t { LIT_RAW = 0, LIT_RLE = 1, LIT_HUF = 2 };

struct EntShared {
    uint32_t lhist[256];
    uint32_t chist[3][64];             // code counts of the LL, OF, ML columns
    int16_t norm[3][64];
    uint16_t stab[3][512];             // FSE encoder: the states of each code, in state order, grouped by code
    int32_t dnb[3][64], dfs[3][64];    // per code: Number_of_Bits transform and offset into stab (zstd's symbolTT)
    uint8_t spread[3][512];            // the code of every state (one table per warp building it)
    uint8_t desc[3][96];
    uint32_t desc_len[3], log[3], mode[3];
    SeqCodes codes;
    // Huffman
    uint32_t hc[256], hw[511];
    uint16_t hparent[511], hcode[256];
    uint8_t horder[256], hdepth[511], hlen[256];
    uint8_t tree[ENT_FSE_TREE_MAX + 1];
    // FSE table of the Huffman weights 0..ENT_HUF_MAXBITS (full-alphabet mode)
    uint32_t whist[ENT_HUF_MAXBITS + 1];
    int16_t wnorm[ENT_HUF_MAXBITS + 1];
    int32_t wdnb[ENT_HUF_MAXBITS + 1], wdfs[ENT_HUF_MAXBITS + 1];
    uint16_t wstab[1 << ENT_WEIGHT_MAXLOG];
    uint8_t wspread[1 << ENT_WEIGHT_MAXLOG];
    uint32_t wsum[ENT_WRITERS / 32], sbits[4];
    uint8_t seqhdr[8];
    uint32_t kind, top, nh, maxlen, tree_len, t1, hs, bitlen, take, co, seqpos, seqhdr_len;
};

__device__ __forceinline__ void writers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(ENT_WRITERS) : "memory"); }

// exclusive prefix sum over the writer threads; *total = the sum of all
__device__ uint32_t writers_scan(uint32_t v, uint32_t *wsum, uint32_t *total) {
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(~0u, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    if (lane == 31) wsum[w] = x;
    writers_sync();
    uint32_t before = 0, all = 0;
    for (uint32_t k = 0; k < ENT_WRITERS / 32; k++) { before += k < w ? wsum[k] : 0; all += wsum[k]; }
    writers_sync();   // wsum is reused by the next scan
    *total = all;
    return before + x - v;
}

// Where ent_table puts a table: the normalised counts, the description (at most dcap bytes of it are stored; desc_len
// counts them all), the encoder form (stab, dnb, dfs; spread is scratch) and its mode and accuracy log.
struct EntTableOut {
    int16_t *norm;
    uint8_t *desc;
    uint32_t dcap;
    uint16_t *stab;
    int32_t *dnb, *dfs;
    uint8_t *spread;
    uint32_t *desc_len, *log, *mode;
};

// The table of nsym codes with counts cnt[] over n >= 1 values, accuracy log at most cap: mode, description, accuracy
// log and encoder form.  Used for the LL / OF / ML columns and for the Huffman weights.
__device__ void ent_table(const uint32_t *cnt, int nsym, int cap, uint32_t n, const EntTableOut o) {
    int16_t *norm = o.norm;
    uint8_t *d = o.desc;
    int distinct = 0, one = 0;
    for (int c = 0; c < nsym; c++) if (cnt[c]) { distinct++; one = c; }
    int log = 0;
    if (distinct == 1) {   // RLE_Mode: the code itself; as a table, one state of accuracy log 0
        for (int c = 0; c < nsym; c++) norm[c] = c == one;
        *o.mode = 1; d[0] = (uint8_t)one; *o.desc_len = 1;
    } else {
        // about 4 sequences per state, within [ENT_MIN_LOG, cap], and at least one state per code present
        log = min(cap, max(ENT_MIN_LOG, 32 - __clz(n) - 2));
        while ((1 << log) < distinct) log++;
        const int size = 1 << log;
        // normalisation: max(1, floor(count * 2^log / n)); while the sum is too large, decrement the largest entry
        // (the lowest code on ties); if too small, the entry with the largest count (lowest code on ties) takes the rest
        int sum = 0;
        for (int c = 0; c < nsym; c++) {
            norm[c] = cnt[c] ? (int16_t)max(1u, cnt[c] * (uint32_t)size / n) : 0;
            sum += norm[c];
        }
        while (sum > size) {
            int k = 0;
            for (int c = 1; c < nsym; c++) if (norm[c] > norm[k]) k = c;
            norm[k]--; sum--;
        }
        if (sum < size) {
            int k = 0;
            for (int c = 1; c < nsym; c++) if (cnt[c] > cnt[k]) k = c;
            norm[k] += size - sum;
        }
        // description (RFC 8878 4.1.1): Accuracy_Log - 5, then count + 1 per code in a variable number of bits, a zero
        // count followed by 2-bit repeat flags for the zero counts after it, until the counts reach 2^log
        uint64_t acc = (uint64_t)(log - ENT_MIN_LOG);
        uint32_t na = 4, q = 0;
        auto put = [&](uint32_t v, uint32_t nb) {
            acc |= (uint64_t)v << na;
            na += nb;
            while (na >= 8) { if (q < o.dcap) d[q] = (uint8_t)acc; q++; acc >>= 8; na -= 8; }
        };
        int remaining = size + 1, threshold = size, nbits = log + 1, c = 0;
        bool prev0 = false;
        while (c < nsym && remaining > 1) {
            if (prev0) {
                int start = c;
                while (norm[c] == 0) c++;
                while (c >= start + 3) { start += 3; put(3, 2); }
                put(c - start, 2);
            }
            int v = norm[c++];
            const int mx = 2 * threshold - 1 - remaining;
            remaining -= v;
            v++;
            if (v >= threshold) v += mx;
            put(v, nbits - (v < mx));
            prev0 = v == 1;
            while (remaining < threshold) { nbits--; threshold >>= 1; }
        }
        if (na) { if (q < o.dcap) d[q] = (uint8_t)acc; q++; }
        *o.mode = 2; *o.desc_len = q;
    }
    *o.log = log;
    fse_ctable(norm, nsym, log, o.spread, o.stab, o.dnb, o.dfs);   // no "less than 1" cells
}

// The FSE form of the tree description into s.tree (RFC 8878 4.2.1.2; lane 0 of warp 0): a header byte holding the
// compressed size, the table description of the weights of symbols 0..top-1 (ent_table, accuracy log at most 6), then
// their bitstream with two interleaved states.  The decoder reads state 1's start, then state 2's, and takes a weight
// from state 1, state 2, state 1, ... until a state update reads past the stream's start; so state 1 codes the even
// positions and state 2 the odd ones, and the encoder runs from the last weight to the first.  Each state starts in
// the lowest state of its weight (zstd's FSE_initCState2), where that update reads at least one bit: the update after
// the second-to-last weight must run past the start for the decoder to stop there, and the "no bits written" start of
// the sequence chain (enc[code][0]) reads none when the weight holds more than half the states, as weight 0 often does.
// Returns the form's size with its header byte, or 0 when it is not allowed: fewer than 2 weights, one distinct weight,
// or more than ENT_FSE_TREE_MAX bytes after the header byte.
__device__ uint32_t ent_fse_tree(EntShared &s, uint32_t top, uint32_t mx) {
    auto wt = [&](uint32_t x) -> uint32_t { return s.hlen[x] ? mx + 1 - s.hlen[x] : 0; };
    for (int w = 0; w <= ENT_HUF_MAXBITS; w++) s.whist[w] = 0;
    for (uint32_t x = 0; x < top; x++) s.whist[wt(x)]++;
    int distinct = 0;
    for (int w = 0; w <= ENT_HUF_MAXBITS; w++) distinct += s.whist[w] != 0;
    if (top < 2 || distinct < 2) return 0;
    uint32_t mode, dlen, log;
    ent_table(s.whist, ENT_HUF_MAXBITS + 1, ENT_WEIGHT_MAXLOG, top,
              EntTableOut{s.wnorm, s.tree + 1, ENT_FSE_TREE_MAX, s.wstab, s.wdnb, s.wdfs, s.wspread, &dlen, &log, &mode});
    if (dlen > ENT_FSE_TREE_MAX) return 0;
    const uint32_t size = 1u << log;
    uint32_t X[2];   // state 1, state 2, kept as 2^log + state
    for (uint32_t t = 0; t < 2; t++) {
        const uint32_t c = wt(top - 1 - ((top - 1 - t) & 1));   // the last position of parity t
        uint32_t first = 0;                                      // stab lists each weight's states in state order
        for (uint32_t w = 0; w < c; w++) first += s.wnorm[w];
        X[t] = size + s.wstab[first];
    }
    uint8_t *out = s.tree + 1;
    uint64_t acc = 0;
    uint32_t na = 0, q = dlen;
    auto put = [&](uint32_t v, uint32_t nb) {
        acc |= (uint64_t)v << na;
        na += nb;
        while (na >= 8) { if (q < ENT_FSE_TREE_MAX) out[q] = (uint8_t)acc; q++; acc >>= 8; na -= 8; }
    };
    for (int k = (int)top - 3; k >= 0; k--) {
        const uint32_t t = k & 1, c = wt(k);
        const uint32_t nb = (uint32_t)((int)X[t] + s.wdnb[c]) >> 16;
        put(X[t] & ((1u << nb) - 1), nb);
        X[t] = size + s.wstab[(int)(X[t] >> nb) + s.wdfs[c]];
    }
    put(X[1] - size, log); put(X[0] - size, log); put(1, 1);
    if (na) { if (q < ENT_FSE_TREE_MAX) out[q] = (uint8_t)acc; q++; }
    if (q > ENT_FSE_TREE_MAX) return 0;
    s.tree[0] = (uint8_t)q;
    return 1 + q;
}

// Huffman code of the literals (warp 0): lengths, canonical codes, tree description and the one-stream bit count.
// `full`: the full-alphabet mode, whose tree description may also take the FSE form.
__device__ void ent_huffman(EntShared &s, uint32_t lane, bool full) {
    const uint32_t top = s.top;
    huf_lengths(s.lhist, top + 1, s.nh, ENT_HUF_MAXBITS, lane, s.hc, s.horder, s.hw, s.hparent, s.hdepth, s.hlen, &s.maxlen);
    if (lane) return;
    // canonical codes (RFC 8878 4.2.1.3): in (length descending, symbol ascending) order, consecutive prefixes in units
    // of 2^(maxbits - length)
    const uint32_t mx = s.maxlen;
    uint32_t nxt = 0, t1 = 0;
    for (uint32_t len = mx; len >= 1; len--)
        for (uint32_t x = 0; x <= top; x++)
            if (s.hlen[x] == len) { s.hcode[x] = (uint16_t)(nxt >> (mx - len)); nxt += 1u << (mx - len); }
    // tree description: the smaller of the allowed forms, the direct one on ties; the literals stay raw when neither is.
    // Direct form (top <= 128): 127 + top, then the weights (maxbits + 1 - length, or 0) of symbols 0..top-1, two per
    // byte, the first in the high nibble; the weight of `top` is implied.  The FSE form only in full-alphabet mode.
    const uint32_t dlen = 1 + (top + 1) / 2, flen = full ? ent_fse_tree(s, top, mx) : 0;
    if (top <= ENT_HUF_MAXSYMBOL && (flen == 0 || dlen <= flen)) {
        auto wt = [&](uint32_t x) -> uint32_t { return x < top && s.hlen[x] ? mx + 1 - s.hlen[x] : 0; };
        s.tree[0] = (uint8_t)(127 + top);
        for (uint32_t k = 0; k < top; k += 2) s.tree[1 + k / 2] = (uint8_t)(wt(k) << 4 | wt(k + 1));
        s.tree_len = dlen;
    } else if (flen) {
        s.tree_len = flen;
    } else {
        s.kind = LIT_RAW;
    }
    for (uint32_t x = 0; x <= top; x++) t1 += s.lhist[x] * s.hlen[x];
    s.t1 = t1;
}

// The Huffman literals section into A (writer threads).  Falls back to raw (s.kind) when it is not smaller.
__device__ void ent_literals(EntShared &s, const uint8_t *lit, uint32_t nl, uint8_t *A) {
    const uint32_t tid = threadIdx.x, tl = s.tree_len;
    const uint32_t ns = nl <= 1023 && tl + s.t1 / 8 + 1 <= 1023 ? 1 : 4;
    const uint32_t seg = ns == 1 ? nl : (nl + 3) / 4;
    uint32_t start[4] = {0, 0, 0, 0};
    // stream k holds literals [k * seg, + len) written from the last to the first, so the bit position of a literal
    // is the sum of the code lengths of the literals after it in its stream
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        if (k == ns) break;
        const uint32_t a = k * seg, len = min(nl, a + seg) - a, per = (len + ENT_WRITERS - 1) / ENT_WRITERS;
        const uint32_t r0 = min(tid * per, len), r1 = min(r0 + per, len);
        uint32_t v = 0, tot;
        for (uint32_t r = r0; r < r1; r++) v += s.hlen[lit[a + len - 1 - r]];
        start[k] = writers_scan(v, s.wsum, &tot);
        if (tid == 0) s.sbits[k] = tot;
    }
    writers_sync();
    uint32_t c = tl + (ns == 4 ? 6 : 0);
    for (uint32_t k = 0; k < ns; k++) c += s.sbits[k] / 8 + 1;   // + the end mark
    const uint32_t big = max(nl, c);
    const uint32_t sf = ns == 1 ? 0 : big <= 1023 ? 1 : big <= 16383 ? 2 : 3, hl = sf < 2 ? 3 : sf + 2;
    const uint32_t hs = hl + c, raw = raw_lit_header_len(nl) + nl;
    if (hs >= raw) {
        if (tid == 0) s.kind = LIT_RAW;
        return;
    }
    const uint32_t hdr = hl + tl + (ns == 4 ? 6 : 0);
    uint32_t *A32 = (uint32_t *)A;
    for (uint32_t k = tid; k < (hs + 3) / 4; k += ENT_WRITERS) A32[k] = 0;
    writers_sync();
    uint32_t pos = hdr;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        if (k == ns) break;
        const uint32_t a = k * seg, len = min(nl, a + seg) - a, per = (len + ENT_WRITERS - 1) / ENT_WRITERS;
        const uint32_t r0 = min(tid * per, len), r1 = min(r0 + per, len);
        const uint32_t bit = pos * 8 + start[k];
        if (r0 < r1) {
            uint32_t w = bit >> 5, na = bit & 31;
            uint64_t acc = 0;
            for (uint32_t r = r0; r < r1; r++) {
                const uint32_t x = lit[a + len - 1 - r];
                acc |= (uint64_t)s.hcode[x] << na;
                na += s.hlen[x];
                if (na >= 32) { atomicOr(A32 + w, (uint32_t)acc); acc >>= 32; na -= 32; w++; }
            }
            if (na) atomicOr(A32 + w, (uint32_t)acc);
        }
        const uint32_t end = pos * 8 + s.sbits[k];
        if (tid == 0) atomicOr(A32 + (end >> 5), 1u << (end & 31));
        pos += s.sbits[k] / 8 + 1;
    }
    writers_sync();
    if (tid == 0) {
        const uint64_t h = 2 | sf << 2 | (uint64_t)nl << 4 | (uint64_t)c << (sf < 2 ? 14 : sf == 2 ? 18 : 22);
        for (uint32_t k = 0; k < hl; k++) A[k] = (uint8_t)(h >> (8 * k));
        for (uint32_t k = 0; k < tl; k++) A[hl + k] = s.tree[k];
        for (uint32_t k = 0; ns == 4 && k < 3; k++) {
            const uint32_t b = s.sbits[k] / 8 + 1;
            A[hl + tl + 2 * k] = (uint8_t)b; A[hl + tl + 2 * k + 1] = (uint8_t)(b >> 8);
        }
        s.hs = hs;
    }
}

template <bool FULL>
__global__ void __launch_bounds__(ENT_THREADS) k_ent_encode(const LzTables *tab, const uint32_t *size, uint64_t first,
                                                            uint8_t *slots, const uint64_t *seqs, const uint32_t *nseq,
                                                            const uint32_t *nlit, uint32_t *info, uint8_t *scratch) {
    __shared__ EntShared s;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t g = first + blockIdx.x;
    const uint32_t n = nseq[g], nl = nlit[g];
    uint8_t *slot = slots + g * LZ_SLOT;
    const uint8_t *lit = slot + 3;
    const uint64_t *sq = seqs + (uint64_t)blockIdx.x * LZ_MAX_SEQ;
    uint8_t *A = scratch + (uint64_t)blockIdx.x * ENT_SCRATCH, *B = A + LZ_SLOT;

    for (uint32_t k = tid; k < 256; k += ENT_THREADS) { s.lhist[k] = 0; s.hlen[k] = 0; }
    for (uint32_t k = tid; k < 3 * 64; k += ENT_THREADS) s.chist[k / 64][k % 64] = 0;
    // field by field: with a copy in 4- or 16-byte words ptxas gives the kernel 48 registers (5 CTAs per SM, not 6)
    for (uint32_t k = tid; k < 128; k += ENT_THREADS) {
        if (k < 36) { s.codes.ll_base[k] = __ldg(&tab->codes.ll_base[k]); s.codes.ll_bits[k] = __ldg(&tab->codes.ll_bits[k]); }
        if (k < 53) { s.codes.ml_base[k] = __ldg(&tab->codes.ml_base[k]); s.codes.ml_bits[k] = __ldg(&tab->codes.ml_bits[k]); }
        if (k < 64) s.codes.ll_code[k] = __ldg(&tab->codes.ll_code[k]);
        s.codes.ml_code[k] = __ldg(&tab->codes.ml_code[k]);
    }
    __syncthreads();
    for (uint32_t i = tid; i < nl; i += ENT_THREADS) atomicAdd(&s.lhist[lit[i]], 1u);
    for (uint32_t k = tid; k < n; k += ENT_THREADS) {
        const Seq q(sq[k], s.codes);
        atomicAdd(&s.chist[0][q.lc], 1u); atomicAdd(&s.chist[1][q.oc], 1u); atomicAdd(&s.chist[2][q.mc], 1u);
    }
    __syncthreads();
    if (warp == 0) {
        uint32_t cnt = 0, top = 0;
        for (uint32_t x = lane; x < 256; x += 32) if (s.lhist[x]) { cnt++; top = x; }
        cnt = __reduce_add_sync(~0u, cnt);
        top = __reduce_max_sync(~0u, top);
        const uint32_t kind = nl == 0 ? LIT_RAW : cnt == 1 ? LIT_RLE : !FULL && top > ENT_HUF_MAXSYMBOL ? LIT_RAW : LIT_HUF;
        if (lane == 0) { s.kind = kind; s.top = top; s.nh = cnt; }
        __syncwarp();
        if (kind == LIT_HUF) ent_huffman(s, lane, FULL);
    } else if (warp <= 3 && lane == 0 && n) {
        const int t = warp - 1;   // LL, OF, ML
        ent_table(s.chist[t], t == 0 ? 36 : t == 1 ? 32 : 53, t == 0 ? ENT_LL_MAXLOG : t == 1 ? ENT_OF_MAXLOG : ENT_ML_MAXLOG,
                  n, EntTableOut{s.norm[t], s.desc[t], sizeof s.desc[t], s.stab[t], s.dnb[t], s.dfs[t], s.spread[t],
                                 &s.desc_len[t], &s.log[t], &s.mode[t]});
    }
    __syncthreads();
    if (warp == ENT_WRITERS / 32) {
        if (lane == 0 && n) {
            LzBits w{B, 0};
            const FseCTable t[3] = {{s.stab[0], s.dnb[0], s.dfs[0], s.log[0]}, {s.stab[1], s.dnb[1], s.dfs[1], s.log[1]},
                                    {s.stab[2], s.dnb[2], s.dfs[2], s.log[2]}};
            seq_bitstream(sq, n, s.codes, t, w);
            s.bitlen = w.q;
        }
    } else if (s.kind == LIT_HUF) {
        ent_literals(s, lit, nl, A);
    }
    __syncthreads();
    if (tid == 0) {
        const uint32_t hl = raw_lit_header_len(nl), kind = s.kind;
        const uint32_t litlen = kind == LIT_HUF ? s.hs : kind == LIT_RLE ? hl + 1 : hl + nl;
        uint32_t q = seq_count_header(n, s.seqhdr), seqlen = 1;
        if (n) {
            s.seqhdr[q++] = (uint8_t)(s.mode[0] << 6 | s.mode[1] << 4 | s.mode[2] << 2);   // LL, OF, ML
            seqlen = q + s.desc_len[0] + s.desc_len[1] + s.desc_len[2] + s.bitlen;
        }
        const uint32_t E = litlen + seqlen, K = info[g] & 0x3FFFFFFFu;   // K9b wins ties
        s.take = E < K && E < size[g];
        s.seqhdr_len = q;
        s.co = kind == LIT_HUF ? 0 : 3 - hl;
        s.seqpos = s.co + litlen;
        if (s.take) {
            info[g] = E | s.co << 30;
            if (kind == LIT_RLE) slot[s.co] |= 1;   // K9b's raw header with Literals_Block_Type 1; slot + 3 holds the value
        }
    }
    __syncthreads();
    if (!s.take) return;
    if (s.kind == LIT_HUF)
        for (uint32_t i = tid; i < s.hs; i += ENT_THREADS) slot[i] = A[i];
    const uint32_t h = s.seqhdr_len, d0 = h + (n ? s.desc_len[0] : 0), d1 = d0 + (n ? s.desc_len[1] : 0);
    const uint32_t d2 = d1 + (n ? s.desc_len[2] : 0), end = d2 + (n ? s.bitlen : 0);
    uint8_t *out = slot + s.seqpos;
    for (uint32_t i = tid; i < end; i += ENT_THREADS)
        out[i] = i < h ? s.seqhdr[i] : i < d0 ? s.desc[0][i - h] : i < d1 ? s.desc[1][i - d0] : i < d2 ? s.desc[2][i - d1] : B[i - d2];
}

cudaError_t launch_ent_encode(const LzTables *tab, const uint32_t *size, uint64_t first, uint32_t nb, uint8_t *slots,
                              const uint64_t *seqs, const uint32_t *nseq, const uint32_t *nlit, uint32_t *info,
                              uint8_t *scratch, bool full, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    if (full) k_ent_encode<true><<<nb, ENT_THREADS, 0, st>>>(tab, size, first, slots, seqs, nseq, nlit, info, scratch);
    else k_ent_encode<false><<<nb, ENT_THREADS, 0, st>>>(tab, size, first, slots, seqs, nseq, nlit, info, scratch);
    return cudaGetLastError();
}

}  // namespace pbsgpu
