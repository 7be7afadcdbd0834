// f3, read side: K13, the zstd decoder of pbsgpu_blob_decode_batch (sm_90a).
//
// One warp per blob, one blob per CTA.  The warp checks the blob's magic and K6's CRC of the payload, then walks its
// frames (RFC 8878 3.1.1) and blocks in order and writes the chunk to its output:
//   Raw / RLE blocks      copied / filled by the 32 lanes
//   literals              Raw: read in place; RLE: filled into the warp's literal slot; Compressed / Treeless: the
//                         Huffman table in shared memory (lane 0 reads the tree description, the lanes fill the table),
//                         then one lane per stream (1 or 4) decodes into the slot
//   sequences             the LL / OF / ML tables in shared memory (Predefined from ZdecTables, RLE, FSE_Compressed read
//                         by lane 0, or Repeat: the table stays); then every lane runs the same FSE chain over the
//                         bitstream (the same loads and the same branches, so no broadcast is needed), resolves the
//                         repeat offsets, and the lanes copy the literals and the match of each sequence
//   checksum              XXH64 of the frame's content (low 32 bits), computed alike by every lane
// Everything a lane reads lies inside [src, src + len) of its blob, its literal slot, its chunk's output written so far
// or its shared memory; every loop is bounded by the format (sizes, counts of at most 2^17 sequences, symbol limits),
// so hostile input ends in a status.  Tables that persist between blocks (Treeless literals, Repeat_Mode) live in the
// CTA's shared memory for the whole frame.
#include <cstring>

#include "internal.cuh"

namespace pbsgpu {

namespace {

constexpr uint32_t HUF_MAXLOG = 11;                 // longest Huffman code RFC 8878 allows
constexpr uint32_t BLOCK_MAX = ZFRAME_BLOCK;        // 128 KiB
// The largest Window_Size upstream's decoder reads: libzstd's streaming decoder refuses a frame that needs more than
// 2^windowLogMax + 1 bytes of window, and windowLogMax is 27 by default.  A Single_Segment frame's window is its content.
constexpr uint64_t WINDOW_MAX = (1ull << 27) + 1;
__device__ __forceinline__ int tab_maxlog(int c) { return c == 1 ? ENT_OF_MAXLOG : ENT_LL_MAXLOG; }   // LL, OF, ML
__device__ __forceinline__ int tab_maxsym(int c) { return c == 0 ? 35 : c == 1 ? 31 : 52; }

struct Shared {
    uint32_t fse[3][512];              // LL, OF, ML decoding tables (fse_dentry)
    uint32_t wdt[64];                  // FSE table of the Huffman weights
    uint16_t huf[1 << HUF_MAXLOG];     // Huffman decoding table: symbol | bits << 8
    uint16_t next[64];
    int16_t norm[64];
    uint8_t spread[512];
    uint8_t w[256];                    // Huffman weights
    uint16_t hpos[256];                // first entry of each symbol in huf
    uint32_t rank[HUF_MAXLOG + 2];     // symbols per weight, then the first entry per weight
    SeqCodes codes;
    int32_t res[4];                    // lane 0's results, read by the warp after __syncwarp
};

__device__ __forceinline__ uint32_t hb32(uint32_t x) { return 31 - __clz(x); }
__device__ __forceinline__ uint32_t le32(const uint8_t *p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }

// Backward bitstream over p[0, n) (RFC 8878 4.1): the highest set bit of p[n - 1] marks its end.  `bit` counts the bits
// not read yet; reads past the start give zeros and drive it negative.
struct BitR {
    const uint8_t *p;
    uint32_t n;
    int64_t bit, wlo;
    uint64_t win;   // bits [wlo, wlo + 64) of the stream
    __device__ bool init(const uint8_t *q, uint32_t len) {
        p = q; n = len; wlo = -1; win = 0; bit = 0;
        if (len == 0 || q[len - 1] == 0) return false;
        bit = 8 * (int64_t)(len - 1) + hb32(q[len - 1]);
        return true;
    }
    // bits [lo, lo + nb) of the stream, nb <= 32; those below bit 0 are zeros
    __device__ uint32_t get(int64_t lo, uint32_t nb) {
        if (nb == 0 || lo + nb <= 0) return 0;
        uint32_t shift = 0;
        if (lo < 0) { shift = (uint32_t)-lo; nb -= shift; lo = 0; }
        if (wlo < 0 || lo < wlo || lo + nb > wlo + 64) {
            int64_t wb = ((lo + nb + 7) >> 3) - 8;
            if (wb < 0) wb = 0;
            win = 0;
            for (int k = 0; k < 8; k++) if ((uint64_t)wb + k < n) win |= (uint64_t)p[wb + k] << (8 * k);
            wlo = wb * 8;
        }
        return (uint32_t)((win >> (lo - wlo)) & ((1ull << nb) - 1)) << shift;
    }
    __device__ uint32_t read(uint32_t nb) { bit -= nb; return get(bit, nb); }
    __device__ uint32_t peek(uint32_t nb) { return get(bit - nb, nb); }
};

// Forward bits of an FSE table description; bytes at or beyond n read as zeros (the caller checks the size used)
struct BitF {
    const uint8_t *p;
    uint32_t n;
    uint64_t pos;
    __device__ uint32_t peek(uint32_t nb) const {   // nb <= 16
        const uint64_t b = pos >> 3;
        uint32_t v = 0;
        for (int k = 0; k < 3; k++) if (b + k < n) v |= (uint32_t)p[b + k] << (8 * k);
        return (v >> (pos & 7)) & ((1u << nb) - 1);
    }
    __device__ uint32_t read(uint32_t nb) { const uint32_t v = peek(nb); pos += nb; return v; }
};

// An FSE table description (RFC 8878 4.1.1) at p[0, n): norm[0, *nsym), *log.  Returns its size in bytes, or -1 when it
// is invalid (accuracy log above maxlog, a code above maxsym, counts that do not sum to 2^log, more bytes than n).
__device__ int read_ncount(const uint8_t *p, uint32_t n, int maxlog, int maxsym, int16_t *norm, int *nsym, int *log) {
    BitF f{p, n, 0};
    const int al = (int)f.read(4) + 5;
    if (al > maxlog) return -1;
    int remaining = (1 << al) + 1, threshold = 1 << al, nbits = al + 1, c = 0;
    bool prev0 = false;
    while (remaining > 1) {
        if (prev0) {   // 2-bit repeat flags: 3 means three more zero counts and another flag
            int n0 = c;
            for (;;) {
                const uint32_t r = f.read(2);
                n0 += (int)r;
                if (n0 > maxsym) return -1;
                if (r != 3) break;
            }
            while (c < n0) norm[c++] = 0;
        }
        if (c > maxsym) return -1;
        const int max = 2 * threshold - 1 - remaining;
        const uint32_t v = f.peek((uint32_t)nbits);
        int count;
        if ((int)(v & (threshold - 1)) < max) { count = (int)(v & (threshold - 1)); f.pos += nbits - 1; }
        else { count = (int)(v & (2 * threshold - 1)); if (count >= threshold) count -= max; f.pos += nbits; }
        count--;   // -1: "less than 1"
        remaining -= count < 0 ? -count : count;
        norm[c++] = (int16_t)count;
        prev0 = count == 0;
        if (remaining < 1) return -1;
        while (remaining < threshold) { nbits--; threshold >>= 1; }
    }
    if (remaining != 1 || f.pos > 8ull * n) return -1;
    *nsym = c; *log = al;
    return (int)((f.pos + 7) >> 3);
}

// Lane 0: the Huffman weights of a Huffman_Tree_Description at p[0, n) into sh.w (the last, implied one included).
// Returns description size | symbols << 8 | table log << 20, or -1.
__device__ int read_weights(Shared &sh, const uint8_t *p, uint32_t n) {
    if (n < 1) return -1;
    const uint32_t hb = p[0];
    uint32_t nw = 0, size;
    if (hb < 128) {   // FSE-compressed weights: two interleaved states over one backward bitstream
        size = 1 + hb;
        if (size > n) return -1;
        int nsym, al;
        const int dl = read_ncount(p + 1, hb, 6, 15, sh.norm, &nsym, &al);
        if (dl < 0) return -1;
        fse_dtable(sh.norm, nsym, al, sh.spread, sh.next, sh.wdt);
        BitR r;
        if (!r.init(p + 1 + dl, hb - (uint32_t)dl)) return -1;
        uint32_t s1 = r.read((uint32_t)al), s2 = r.read((uint32_t)al);
        for (;;) {   // at most 255 weights
            if (nw > 253) return -1;
            uint32_t e = sh.wdt[s1];
            sh.w[nw++] = (uint8_t)e;
            s1 = (e >> 16) + r.read((e >> 8) & 0xFF);
            if (r.bit < 0) { sh.w[nw++] = (uint8_t)sh.wdt[s2]; break; }
            if (nw > 253) return -1;
            e = sh.wdt[s2];
            sh.w[nw++] = (uint8_t)e;
            s2 = (e >> 16) + r.read((e >> 8) & 0xFF);
            if (r.bit < 0) { sh.w[nw++] = (uint8_t)sh.wdt[s1]; break; }
        }
    } else {          // direct: 4 bits per weight
        nw = hb - 127;
        size = 1 + (nw + 1) / 2;
        if (size > n) return -1;
        for (uint32_t k = 0; k < nw; k++) sh.w[k] = (uint8_t)(k & 1 ? p[1 + k / 2] & 15 : p[1 + k / 2] >> 4);
    }
    uint32_t total = 0;
    for (uint32_t k = 0; k < nw; k++) {
        if (sh.w[k] > HUF_MAXLOG) return -1;
        if (sh.w[k]) total += 1u << (sh.w[k] - 1);
    }
    if (total == 0) return -1;
    const uint32_t log = hb32(total) + 1, rest = (1u << log) - total;
    if (log > HUF_MAXLOG || (rest & (rest - 1))) return -1;
    sh.w[nw] = (uint8_t)(hb32(rest) + 1);
    uint32_t ones = 0;
    for (uint32_t k = 0; k <= nw; k++) ones += sh.w[k] == 1;
    if (ones < 2 || (ones & 1)) return -1;   // a complete prefix code has an even number of longest codes
    return (int)(size | (nw + 1) << 8 | log << 20);
}

// The warp: the Huffman decoding table of nsym weights sh.w at log `log` (zstd's HUF_readDTableX1 order: by weight,
// then by symbol).  Lane 0 places the symbols, the lanes fill their entries.
__device__ __forceinline__ void fill_huf(Shared &sh, uint32_t nsym, uint32_t log, uint32_t lane) {
    if (lane == 0) {
        for (uint32_t w = 0; w <= HUF_MAXLOG + 1; w++) sh.rank[w] = 0;
        for (uint32_t s = 0; s < nsym; s++) sh.rank[sh.w[s]]++;
        for (uint32_t w = 1, pos = 0; w <= log; w++) { const uint32_t c = sh.rank[w]; sh.rank[w] = pos; pos += c << (w - 1); }
        for (uint32_t s = 0; s < nsym; s++) {
            const uint32_t w = sh.w[s];
            if (w) { sh.hpos[s] = (uint16_t)sh.rank[w]; sh.rank[w] += 1u << (w - 1); }
        }
    }
    __syncwarp();
    for (uint32_t s = 0; s < nsym; s++) {
        const uint32_t w = sh.w[s];
        if (!w) continue;
        const uint32_t len = 1u << (w - 1), at = sh.hpos[s];
        for (uint32_t k = lane; k < len; k += 32) sh.huf[at + k] = (uint16_t)(s | (log + 1 - w) << 8);
    }
    __syncwarp();
}

// One lane: cnt symbols of the Huffman stream p[0, n) into dst; false unless the stream is consumed exactly
__device__ __forceinline__ bool huf_stream(const uint16_t *huf, uint32_t log, const uint8_t *p, uint32_t n, uint8_t *dst, uint32_t cnt) {
    BitR r;
    if (!r.init(p, n)) return false;
    for (uint32_t k = 0; k < cnt; k++) {
        const uint32_t e = huf[r.peek(log)];
        dst[k] = (uint8_t)e;
        r.bit -= e >> 8;
    }
    return r.bit == 0;
}

// What a frame carries from block to block
struct Frame {
    uint8_t *out;
    uint64_t cap, fstart, pos;   // output capacity, start of this frame's content, bytes written
    uint32_t bmax;               // Block_Maximum_Size
    uint32_t rep0, rep1, rep2;
    uint32_t hlog, log[3];
    bool have_huf, have[3];
};

enum : int32_t { ST_OK = PBSGPU_DEC_OK, ST_FRAME = PBSGPU_DEC_BAD_FRAME, ST_SIZE = PBSGPU_DEC_BAD_SIZE };

// The Literals_Section at p[0, n): the literals at *lit (in place or in slot), *nlit of them.  Returns its size, or -1.
__device__ __forceinline__ int read_literals(Shared &sh, Frame &f, const uint8_t *p, uint32_t n, uint8_t *slot, uint32_t lane,
                             const uint8_t **lit, uint32_t *nlit) {
    if (n < 1) return -1;
    const uint32_t t = p[0] & 3, sf = (p[0] >> 2) & 3;
    if (t < 2) {   // Raw / RLE
        uint32_t lh, size;
        if ((sf & 1) == 0) { lh = 1; size = p[0] >> 3; }
        else if (sf == 1) { lh = 2; if (n < 2) return -1; size = (p[0] >> 4) + ((uint32_t)p[1] << 4); }
        else { lh = 3; if (n < 3) return -1; size = (p[0] >> 4) + ((uint32_t)p[1] << 4) + ((uint32_t)p[2] << 12); }
        if (size > f.bmax) return -1;
        *nlit = size;
        if (t == 0) {
            if (lh + size > n) return -1;
            *lit = p + lh;
            return (int)(lh + size);
        }
        if (lh + 1 > n) return -1;
        const uint8_t v = p[lh];
        for (uint32_t k = lane; k < size; k += 32) slot[k] = v;
        __syncwarp();
        *lit = slot;
        return (int)(lh + 1);
    }
    // Compressed / Treeless: sizes of 10, 10, 14 or 18 bits; one stream with Size_Format 00, else four
    const uint32_t lh = sf < 2 ? 3 : sf + 2, bits = sf < 2 ? 10 : sf == 2 ? 14 : 18;
    if (n < lh) return -1;
    uint64_t h = 0;
    for (uint32_t k = 0; k < lh; k++) h |= (uint64_t)p[k] << (8 * k);
    const uint32_t regen = (uint32_t)(h >> 4) & ((1u << bits) - 1), csize = (uint32_t)(h >> (4 + bits)) & ((1u << bits) - 1);
    const bool four = sf != 0;
    if (regen > f.bmax || lh + csize > n || (four && regen < 6)) return -1;
    const uint8_t *q = p + lh;
    uint32_t qn = csize;
    if (t == 2) {
        if (lane == 0) sh.res[0] = read_weights(sh, q, qn);
        __syncwarp();
        const int r = sh.res[0];
        if (r < 0) return -1;
        const uint32_t tl = (uint32_t)r & 0xFF;
        f.hlog = (uint32_t)r >> 20;
        fill_huf(sh, ((uint32_t)r >> 8) & 0xFFF, f.hlog, lane);
        f.have_huf = true;
        q += tl; qn -= tl;
    } else if (!f.have_huf) {
        return -1;
    }
    uint32_t so = 0, sl = qn, dofs = 0, dcnt = regen;   // this lane's stream
    const uint32_t ns = four ? 4 : 1;
    if (four) {
        if (qn < 6) return -1;
        const uint32_t l1 = q[0] | q[1] << 8, l2 = q[2] | q[3] << 8, l3 = q[4] | q[5] << 8;
        if ((uint64_t)l1 + l2 + l3 > qn - 6) return -1;
        const uint32_t seg = (regen + 3) / 4, k = lane < 4 ? lane : 0;
        so = 6 + (k > 0 ? l1 : 0) + (k > 1 ? l2 : 0) + (k > 2 ? l3 : 0);
        sl = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : qn - 6 - l1 - l2 - l3;
        dofs = seg * k;
        dcnt = k < 3 ? seg : regen - 3 * seg;
    }
    bool ok = true;
    if (lane < ns) ok = huf_stream(sh.huf, f.hlog, q + so, sl, slot + dofs, dcnt);
    if (!__all_sync(~0u, ok)) return -1;
    __syncwarp();
    *lit = slot;
    *nlit = regen;
    return (int)(lh + csize);
}

// The table of column c (LL, OF, ML) in `mode` at p[0, n).  Returns its description size, or -1.
__device__ __forceinline__ int read_table(Shared &sh, const ZdecTables &T, Frame &f, int c, uint32_t mode, const uint8_t *p, uint32_t n,
                          uint32_t lane) {
    if (mode == 3) return f.have[c] ? 0 : -1;   // Repeat_Mode
    f.have[c] = true;
    if (mode == 0) {
        const uint32_t *src = c == 0 ? T.ll_dt : c == 1 ? T.of_dt : T.ml_dt;
        const uint32_t size = c == 1 ? 32 : 64;
        for (uint32_t k = lane; k < size; k += 32) sh.fse[c][k] = src[k];
        __syncwarp();
        f.log[c] = c == 1 ? 5 : 6;
        return 0;
    }
    if (mode == 1) {
        if (n < 1 || p[0] > tab_maxsym(c)) return -1;
        if (lane == 0) sh.fse[c][0] = fse_dentry(p[0], 0, 0);
        __syncwarp();
        f.log[c] = 0;
        return 1;
    }
    if (lane == 0) {
        int nsym, al;
        const int dl = read_ncount(p, n, tab_maxlog(c), tab_maxsym(c), sh.norm, &nsym, &al);
        if (dl >= 0) fse_dtable(sh.norm, nsym, al, sh.spread, sh.next, sh.fse[c]);
        sh.res[1] = dl; sh.res[2] = al;
    }
    __syncwarp();
    const int dl = sh.res[1];
    f.log[c] = (uint32_t)sh.res[2];
    __syncwarp();
    return dl;
}

__device__ __forceinline__ void copy_bytes(uint8_t *dst, const uint8_t *src, uint32_t n, uint32_t lane) {
    for (uint32_t k = lane; k < n; k += 32) dst[k] = src[k];
}

// A Compressed_Block's content at p[0, n)
__device__ __forceinline__ int32_t decode_block(Shared &sh, const ZdecTables &T, Frame &f, const uint8_t *p, uint32_t n, uint8_t *slot,
                                uint32_t lane) {
    const uint8_t *lit;
    uint32_t nlit;
    const int used = read_literals(sh, f, p, n, slot, lane, &lit, &nlit);
    if (used < 0) return ST_FRAME;
    p += used; n -= (uint32_t)used;
    if (n < 1) return ST_FRAME;
    uint32_t nseq = p[0], h = 1;
    if (nseq == 0) { if (n != 1) return ST_FRAME; }
    else if (nseq == 255) { if (n < 3) return ST_FRAME; nseq = p[1] + ((uint32_t)p[2] << 8) + 0x7F00; h = 3; }
    else if (nseq >= 128) { if (n < 2) return ST_FRAME; nseq = ((nseq - 128) << 8) + p[1]; h = 2; }
    p += h; n -= h;
    const uint64_t b0 = f.pos;
    uint32_t lpos = 0;
    if (nseq) {
        if (n < 1 || (p[0] & 3)) return ST_FRAME;
        const uint32_t modes = p[0];
        p++; n--;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const int dl = read_table(sh, T, f, c, (modes >> (6 - 2 * c)) & 3, p, n, lane);
            if (dl < 0) return ST_FRAME;
            p += dl; n -= (uint32_t)dl;
        }
        BitR r;
        if (!r.init(p, n)) return ST_FRAME;
        const SeqCodes &sc = sh.codes;
        const uint32_t *tl = sh.fse[0], *to = sh.fse[1], *tm = sh.fse[2];
        uint32_t sl = r.read(f.log[0]), so = r.read(f.log[1]), sm = r.read(f.log[2]);
        for (uint32_t k = 0; k < nseq; k++) {
            const uint32_t el = tl[sl], eo = to[so], em = tm[sm];
            const uint32_t oc = eo & 0xFF, mc = em & 0xFF, lc = el & 0xFF;
            const uint32_t ov = (1u << oc) + r.read(oc);
            const uint32_t ml = sc.ml_base[mc] + r.read(sc.ml_bits[mc]);
            const uint32_t ll = sc.ll_base[lc] + r.read(sc.ll_bits[lc]);
            if (k + 1 < nseq) {
                sl = (el >> 16) + r.read((el >> 8) & 0xFF);
                sm = (em >> 16) + r.read((em >> 8) & 0xFF);
                so = (eo >> 16) + r.read((eo >> 8) & 0xFF);
            }
            uint32_t off;   // RFC 8878 3.1.1.5
            if (ov > 3) {
                off = ov - 3;
                f.rep2 = f.rep1; f.rep1 = f.rep0; f.rep0 = off;
            } else {
                const uint32_t idx = ov - 1 + (ll == 0);
                if (idx == 0) off = f.rep0;
                else {
                    off = idx == 1 ? f.rep1 : idx == 2 ? f.rep2 : f.rep0 - 1;
                    if (idx >= 2) f.rep2 = f.rep1;
                    f.rep1 = f.rep0; f.rep0 = off;
                }
            }
            if ((uint64_t)lpos + ll > nlit || f.pos + ll + ml - b0 > f.bmax) return ST_FRAME;
            if (off == 0 || off > f.pos + ll - f.fstart) return ST_FRAME;
            if (f.pos + ll + ml > f.cap) return ST_SIZE;
            uint8_t *d = f.out + f.pos;
            copy_bytes(d, lit + lpos, ll, lane);
            __syncwarp();
            d += ll;
            const uint8_t *s = d - off;
            if (off >= ml) copy_bytes(d, s, ml, lane);
            else for (uint32_t j = lane; j < ml; j += 32) d[j] = s[j % off];
            __syncwarp();
            f.pos += ll + ml;
            lpos += ll;
        }
        if (r.bit != 0) return ST_FRAME;
    }
    const uint32_t rest = nlit - lpos;
    if (f.pos + rest - b0 > f.bmax) return ST_FRAME;
    if (f.pos + rest > f.cap) return ST_SIZE;
    copy_bytes(f.out + f.pos, lit + lpos, rest, lane);
    __syncwarp();
    f.pos += rest;
    return ST_OK;
}

// XXH64 (seed 0) of p[0, n)
__device__ __forceinline__ uint64_t xxh64(const uint8_t *p, uint64_t n) {
    constexpr uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull,
                       P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    auto rotl = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
    auto round = [&](uint64_t acc, uint64_t v) { acc += v * P2; acc = rotl(acc, 31); return acc * P1; };
    const bool aligned = ((uintptr_t)p & 7) == 0;
    auto ld64 = [&](uint64_t i) {
        if (aligned) return *(const uint64_t *)(p + i);
        uint64_t v = 0;
        for (int k = 0; k < 8; k++) v |= (uint64_t)p[i + k] << (8 * k);
        return v;
    };
    uint64_t i = 0, h;
    if (n >= 32) {
        uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        for (; i + 32 <= n; i += 32) {
            v1 = round(v1, ld64(i)); v2 = round(v2, ld64(i + 8)); v3 = round(v3, ld64(i + 16)); v4 = round(v4, ld64(i + 24));
        }
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        h ^= round(0, v1); h = h * P1 + P4;
        h ^= round(0, v2); h = h * P1 + P4;
        h ^= round(0, v3); h = h * P1 + P4;
        h ^= round(0, v4); h = h * P1 + P4;
    } else {
        h = P5;
    }
    h += n;
    for (; i + 8 <= n; i += 8) { h ^= round(0, ld64(i)); h = rotl(h, 27) * P1 + P4; }
    if (i + 4 <= n) { h ^= (uint64_t)le32(p + i) * P1; h = rotl(h, 23) * P2 + P3; i += 4; }
    for (; i < n; i++) { h ^= p[i] * P5; h = rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// The frames of a compressed payload p[0, n) into out[0, cap)
__device__ __forceinline__ int32_t decode_frames(Shared &sh, const ZdecTables &T, const uint8_t *p, uint64_t n, uint8_t *out, uint64_t cap,
                                 uint8_t *slot, uint32_t lane) {
    Frame f;
    f.out = out; f.cap = cap; f.pos = 0;
    bool bad_checksum = false;
    uint64_t q = 0;
    while (q < n) {   // every frame consumes at least 4 bytes
        if (n - q < 4) return ST_FRAME;
        const uint32_t magic = le32(p + q);
        if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {   // skippable frame
            if (n - q < 8) return ST_FRAME;
            const uint32_t sz = le32(p + q + 4);
            if (sz > n - q - 8) return ST_FRAME;
            q += 8 + (uint64_t)sz;
            continue;
        }
        if (magic != 0xFD2FB528u) return ST_FRAME;
        q += 4;
        if (q >= n) return ST_FRAME;
        const uint32_t fhd = p[q++];
        const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
        if (fhd & 8) return ST_FRAME;   // reserved bit
        uint64_t window = 0;
        if (!single) {
            if (q >= n) return ST_FRAME;
            const uint32_t wd = p[q++], wlog = 10 + (wd >> 3);
            window = (1ull << wlog) + ((1ull << wlog) >> 3) * (wd & 7);
        }
        const uint32_t did_size = did_flag == 3 ? 4 : did_flag;
        const uint32_t fcs_size = fcs_flag == 0 ? single : 1u << fcs_flag;
        if (n - q < did_size + fcs_size) return ST_FRAME;
        for (uint32_t k = 0; k < did_size; k++) if (p[q + k]) return ST_FRAME;   // Dictionary_ID 0 only
        q += did_size;
        uint64_t fcs = 0;
        for (uint32_t k = 0; k < fcs_size; k++) fcs |= (uint64_t)p[q + k] << (8 * k);
        if (fcs_size == 2) fcs += 256;
        q += fcs_size;
        if (single) window = fcs;
        if (window > WINDOW_MAX) return ST_FRAME;
        f.bmax = (uint32_t)(window < BLOCK_MAX ? window : BLOCK_MAX);
        f.fstart = f.pos;
        f.rep0 = 1; f.rep1 = 4; f.rep2 = 8;
        f.have_huf = f.have[0] = f.have[1] = f.have[2] = false;
        for (;;) {   // every block consumes at least 3 bytes
            if (n - q < 3) return ST_FRAME;
            const uint32_t bh = p[q] | p[q + 1] << 8 | p[q + 2] << 16, type = (bh >> 1) & 3, bsize = bh >> 3;
            q += 3;
            if (type == 3) return ST_FRAME;
            if (type == 0) {
                if (bsize > f.bmax || bsize > n - q) return ST_FRAME;
                if (f.pos + bsize > cap) return ST_SIZE;
                copy_bytes(out + f.pos, p + q, bsize, lane);
                q += bsize; f.pos += bsize;
            } else if (type == 1) {
                if (bsize > f.bmax || q >= n) return ST_FRAME;
                if (f.pos + bsize > cap) return ST_SIZE;
                const uint8_t v = p[q];
                for (uint32_t k = lane; k < bsize; k += 32) out[f.pos + k] = v;
                q += 1; f.pos += bsize;
            } else {
                if (bsize > f.bmax || bsize > n - q) return ST_FRAME;
                const int32_t r = decode_block(sh, T, f, p + q, bsize, slot, lane);
                if (r != ST_OK) return r;
                q += bsize;
            }
            __syncwarp();
            if (bh & 1) break;
        }
        if (fcs_size && f.pos - f.fstart != fcs) return ST_FRAME;
        if (checksum) {
            if (n - q < 4) return ST_FRAME;
            if ((uint32_t)xxh64(out + f.fstart, f.pos - f.fstart) != le32(p + q)) bad_checksum = true;
            q += 4;
        }
    }
    if (f.pos != cap) return ST_SIZE;
    return bad_checksum ? PBSGPU_DEC_BAD_CHECKSUM : ST_OK;
}

__device__ __constant__ uint8_t MAGICS[4][8] = {
    {66, 171, 56, 7, 190, 131, 112, 161},                  // uncompressed
    {49, 185, 88, 66, 111, 182, 163, 127},                 // zstd compressed
    {0x7b, 0x67, 0x85, 0xbe, 0x22, 0x2d, 0x4c, 0xf0},      // encrypted
    {0xe6, 0x59, 0x1b, 0xbf, 0x0b, 0xbf, 0xd8, 0x0b}};     // encrypted and compressed

__global__ void __launch_bounds__(32) k_zdec(const uint8_t *base, const ZdecBlob *blobs, const uint32_t *crc,
                                             const ZdecTables *tab, uint8_t *lits, int32_t *status) {
    __shared__ Shared sh;
    const uint32_t lane = threadIdx.x, k = blockIdx.x;
    const ZdecBlob b = blobs[k];
    const uint8_t *p = base + b.src;
    uint8_t *out = (uint8_t *)(uintptr_t)b.dst;
    for (uint32_t i = lane; i < sizeof(SeqCodes); i += 32) ((uint8_t *)&sh.codes)[i] = ((const uint8_t *)&tab->codes)[i];
    __syncwarp();
    int32_t st = PBSGPU_DEC_BAD_MAGIC;
    int kind = -1;
    if (b.len >= 12)
        for (int m = 0; m < 4 && kind < 0; m++) {
            bool eq = true;
            for (int j = 0; j < 8; j++) eq &= p[j] == MAGICS[m][j];
            if (eq) kind = m;
        }
    if (kind >= 2) st = PBSGPU_DEC_ENCRYPTED;
    else if (kind >= 0 && le32(p + 8) != crc[k]) st = PBSGPU_DEC_BAD_CRC;
    else if (kind == 0) {
        if (b.len - 12 != b.cap) st = PBSGPU_DEC_BAD_SIZE;
        else { copy_bytes(out, p + 12, (uint32_t)b.cap, lane); st = PBSGPU_DEC_OK; }
    } else if (kind == 1) {
        st = decode_frames(sh, *tab, p + 12, b.len - 12, out, b.cap, lits + (uint64_t)k * ZDEC_LIT_SLOT, lane);
    }
    if (lane == 0) status[k] = st;
}

// one thread per blob: its first min(len, ZDEC_HEAD) bytes to heads + ZDEC_HEAD * i, zeros after them
__global__ void k_blob_heads(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint32_t n, uint8_t *heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t *p = base + off[i];
    const uint64_t l = len[i];
    for (uint32_t j = 0; j < ZDEC_HEAD; j++) heads[(uint64_t)ZDEC_HEAD * i + j] = j < l ? p[j] : 0;
}

// one thread per entry: the 16 bytes at stage + at[k] (16 B aligned)
__global__ void k_stage_heads(uint8_t *stage, const uint64_t *at, const uint4 *head, uint32_t n) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) *(uint4 *)(stage + at[k]) = head[k];
}

}  // namespace

cudaError_t launch_blob_heads(const uint8_t *base, const uint64_t *off, const uint64_t *len, uint32_t n, uint8_t *heads,
                              cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    k_blob_heads<<<(n + 127) / 128, 128, 0, st>>>(base, off, len, n, heads);
    return cudaGetLastError();
}

cudaError_t launch_stage_heads(uint8_t *stage, const uint64_t *at, const void *head, uint32_t n, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    k_stage_heads<<<(n + 127) / 128, 128, 0, st>>>(stage, at, (const uint4 *)head, n);
    return cudaGetLastError();
}

cudaError_t launch_zdec(const uint8_t *base, const ZdecBlob *b, const uint32_t *crc, uint32_t nb, const ZdecTables *tab,
                        uint8_t *lits, int32_t *status, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    k_zdec<<<nb, 32, 0, st>>>(base, b, crc, tab, lits, status);
    return cudaGetLastError();
}

void zdec_fill_tables_host(void *dst) {
    ZdecTables t;
    LzTables lt;
    lz_fill_tables_host(&lt);
    t.codes = lt.codes;
    uint8_t spread[64];
    uint16_t next[53];
    fse_dtable(PREDEF_LL_NORM, 36, 6, spread, next, t.ll_dt);
    fse_dtable(PREDEF_OF_NORM, 29, 5, spread, next, t.of_dt);
    fse_dtable(PREDEF_ML_NORM, 53, 6, spread, next, t.ml_dt);
    memcpy(dst, &t, sizeof t);
}

}  // namespace pbsgpu
