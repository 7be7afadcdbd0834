// pbs_plus_b200/csrc/capi_zip.cu -- C ABI of the zip restore (f3, read side): raw Deflate streams of byte ranges (K9a's
// Deflate parse, or with _lzc K16's hash-chain parse, then K15, deflate.cu), the CRC-32 combination of pieces, and the
// zip container written on the host.
#include <time.h>

#include <algorithm>
#include <cstring>

#include "host.hpp"

using namespace pbsgpu;

extern "C" uint64_t pbsgpu_deflate_bound(uint64_t len) {
    return len + 15 * ((len + DEFLATE_SEGMENT - 1) / DEFLATE_SEGMENT) + 2;
}

// GF(2) polynomial arithmetic modulo the reflected CRC-32 polynomial: a * b, and x^(n * 2^k)
static uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

extern "C" uint32_t pbsgpu_crc32_combine(uint32_t crc1, uint32_t crc2, uint64_t len2) {
    uint32_t sq = 1u << 30, p = 1u << 31;   // x^1; x^0
    for (uint64_t n = len2 * 8; n; n >>= 1) {   // x^(8 len2) by squaring
        if (n & 1) p = multmodp(sq, p);
        sq = multmodp(sq, sq);
    }
    return multmodp(p, crc1) ^ crc2;
}

// lzc: K16's DEFLATE instantiation parses each pass of DCH_PASS_SEGS segments (every segment one chunk of one block of
// ChainArgs) instead of K9a; K15 and the compaction are the same.
static int deflate_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                         const uint8_t *more, uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out,
                         bool lzc) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !out_len))) return PBSGPU_EINVAL;
    Guard g(ctx);
    for (uint32_t i = 0; i < n; i++)
        if (more && more[i] && len[i] % DEFLATE_SEGMENT)
            return fail(ctx, PBSGPU_EINVAL, "range %u: a piece that a later call continues must be a multiple of 128 KiB", i);
    if (n == 0) return PBSGPU_OK;
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    const bool out_dev = pbsgpu_is_device_ptr(out);
    uint32_t *d_crc = nullptr;
    if (crc_out) {
        d_crc = b.get<uint32_t>(n);
        if (!d_crc) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
        if (int rc = pbsgpu_crc32_enqueue(b, dbase, off, len, n, d_crc)) return rc;
    }
    // the segments of every range, in range order
    std::vector<uint64_t> src;
    std::vector<uint32_t> size, range;
    std::vector<uint8_t> fin;
    for (uint32_t i = 0; i < n; i++) {
        out_len[i] = 0;
        const uint64_t ns = (len[i] + DEFLATE_SEGMENT - 1) / DEFLATE_SEGMENT;
        for (uint64_t k = 0; k < ns; k++) {
            src.push_back(off[i] + k * DEFLATE_SEGMENT);
            size.push_back((uint32_t)std::min<uint64_t>(DEFLATE_SEGMENT, len[i] - k * DEFLATE_SEGMENT));
            range.push_back(i);
            fin.push_back(!(more && more[i]) && k + 1 == ns);
        }
    }
    const uint64_t nseg = src.size();
    // the empty final stream: the empty fixed block
    static const uint8_t EMPTY[2] = {0x03, 0x00};
    for (uint32_t i = 0; i < n; i++)
        if (len[i] == 0 && !(more && more[i])) {
            if (out_dev) { if (b.ok()) b.e = cudaMemcpyAsync(out + out_off[i], EMPTY, 2, cudaMemcpyHostToDevice, b.st); }
            else memcpy(out + out_off[i], EMPTY, 2);
            out_len[i] = 2;
        }
    if (nseg) {
        const uint64_t pass = lzc ? DCH_PASS_SEGS : DEFLATE_PASS_SEGS, pcap = std::min<uint64_t>(nseg, pass);
        uint64_t *d_src = b.upload(src.data(), nseg);
        uint32_t *d_size = b.upload(size.data(), nseg);
        uint8_t *d_fin = b.upload(fin.data(), nseg);
        uint8_t *d_lits = b.get<uint8_t>(pcap * LZ_SLOT);
        uint64_t *d_seqs = b.get<uint64_t>(pcap * LZ_MAX_SEQ);
        uint32_t *d_nseq = b.get<uint32_t>(pcap), *d_nlit = b.get<uint32_t>(pcap), *d_len = b.get<uint32_t>(pcap);
        uint8_t *d_out = b.get<uint8_t>(pcap * DEFLATE_SLOT);
        uint8_t *stage = out_dev ? nullptr : b.get<uint8_t>(pcap * DEFLATE_SLOT);
        ReadPiece *d_pieces = b.get<ReadPiece>(pcap);
        uint64_t *d_first = b.get<uint64_t>(pcap + 1);
        if (!d_src || !d_size || !d_fin || !d_lits || !d_seqs || !d_nseq || !d_nlit || !d_len || !d_out ||
            (!out_dev && !stage) || !d_pieces || !d_first)
            return fail(ctx, PBSGPU_ENOMEM, "deflate: device allocation failed");
        // lzc: the segments' sizes as K16 takes them, their first positions in the call, and the scratch of one pass
        std::vector<uint64_t> vfirst, len64;
        uint64_t *d_vfirst = nullptr, *d_len64 = nullptr;
        uint8_t *scratch = nullptr;
        if (lzc) {
            vfirst.assign(nseg + 1, 0);
            len64.assign(size.begin(), size.end());
            for (uint64_t s = 0; s < nseg; s++) vfirst[s + 1] = vfirst[s] + size[s];
            uint64_t most = 0;
            for (uint64_t f = 0; f < nseg; f += pass) most = std::max(most, vfirst[std::min(nseg, f + pass)] - vfirst[f]);
            const size_t sb = chain_scratch_bytes(most);
            d_vfirst = b.upload(vfirst.data(), nseg + 1);
            d_len64 = b.upload(len64.data(), nseg);
            scratch = b.get<uint8_t>(sb);
            if (!d_vfirst || !d_len64 || !scratch)
                return fail(ctx, PBSGPU_ENOMEM, "deflate: chain search scratch of %llu bytes failed", (unsigned long long)sb);
        }
        std::vector<uint32_t> slen(pcap);
        std::vector<ReadPiece> pieces(pcap);
        std::vector<uint64_t> first(pcap + 1);
        struct Run { uint64_t stage, out, len; };
        std::vector<Run> runs;
        for (uint64_t f = 0; f < nseg; f += pass) {
            const uint32_t pn = (uint32_t)std::min<uint64_t>(pass, nseg - f);
            if (lzc) {
                const ChainArgs a{dbase, d_src, d_len64, d_vfirst, (uint32_t)f, (uint32_t)(f + pn), vfirst[f + pn] - vfirst[f],
                                  vfirst[f], d_src, d_vfirst, d_size, f, f + pn};
                if (b.ok()) b.e = launch_chain_search(a, scratch, b.st, true);
                if (b.ok()) b.e = launch_chain_parse(a, scratch, f, pn, d_lits, d_seqs, d_nseq, d_nlit, b.st, true);
            } else if (b.ok()) {
                b.e = launch_lz_parse_deflate(dbase, d_src + f, d_size + f, pn, d_lits, d_seqs, d_nseq, d_nlit, b.st);
            }
            if (b.ok()) b.e = launch_deflate_encode(dbase, d_src + f, d_size + f, d_fin + f, pn, d_lits, d_seqs, d_nseq, d_nlit,
                                                    d_out, d_len, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(slen.data(), d_len, pn * 4ull, cudaMemcpyDeviceToHost, b.st);
            if (int rc = b.finish("deflate encode")) return rc;
            // compaction: each segment behind the earlier ones of its range (K14), through the stage for a host out
            runs.clear();
            uint64_t staged = 0;
            first[0] = 0;
            for (uint32_t s = 0; s < pn; s++) {
                const uint32_t i = range[f + s];
                const uint64_t dst = out_off[i] + out_len[i];
                const uint64_t to = out_dev ? (uint64_t)(uintptr_t)out + dst : (uint64_t)(uintptr_t)stage + staged;
                pieces[s] = {(uint64_t)(uintptr_t)d_out + (uint64_t)s * DEFLATE_SLOT, to, slen[s]};
                first[s + 1] = first[s] + (slen[s] + READ_TILE - 1) / READ_TILE;
                if (!out_dev) {
                    if (!runs.empty() && runs.back().out + runs.back().len == dst) runs.back().len += slen[s];
                    else runs.push_back({staged, dst, slen[s]});
                    staged += slen[s];
                }
                out_len[i] += slen[s];
            }
            if (b.ok()) b.e = cudaMemcpyAsync(d_pieces, pieces.data(), pn * sizeof(ReadPiece), cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(d_first, first.data(), (pn + 1) * 8ull, cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = launch_read_gather(d_pieces, d_first, pn, first[pn], ctx->sm_count, b.st);
            for (const Run &u : runs)
                if (b.ok()) b.e = cudaMemcpyAsync(out + u.out, stage + u.stage, u.len, cudaMemcpyDeviceToHost, b.st);
            if (int rc = b.finish("deflate compaction")) return rc;
        }
    }
    if (crc_out && b.ok()) b.e = cudaMemcpyAsync(crc_out, d_crc, n * 4ull, cudaMemcpyDeviceToHost, b.st);
    return b.finish("deflate batch");
}

extern "C" int pbsgpu_deflate_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                    const uint8_t *more, uint8_t *out, const uint64_t *out_off, uint64_t *out_len,
                                    uint32_t *crc_out) {
    return deflate_batch(ctx, base, off, len, n, more, out, out_off, out_len, crc_out, false);
}

extern "C" int pbsgpu_deflate_batch_lzc(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len,
                                        uint32_t n, const uint8_t *more, uint8_t *out, const uint64_t *out_off,
                                        uint64_t *out_len, uint32_t *crc_out) {
    return deflate_batch(ctx, base, off, len, n, more, out, out_off, out_len, crc_out, true);
}

// ---- the zip container --------------------------------------------------------------------------------------------
namespace {
constexpr uint32_t U32MAX = 0xFFFFFFFFu;
constexpr uint16_t VERSION_20 = 20, VERSION_45 = 45, CREATOR_UNIX = 3 << 8;

struct Put {
    uint8_t *p;
    uint64_t q = 0;
    bool on;
    void u8(uint32_t v) { if (on) p[q] = (uint8_t)v; q++; }
    void u16(uint32_t v) { u8(v); u8(v >> 8); }
    void u32(uint32_t v) { u16(v); u16(v >> 16); }
    void u64(uint64_t v) { u32((uint32_t)v); u32((uint32_t)(v >> 32)); }
    void bytes(const uint8_t *s, uint64_t n) { if (on && n) memcpy(p + q, s, n); q += n; }
};

bool is_dir(const pbsgpu_zip_entry *e) { return e->name_len && e->name[e->name_len - 1] == '/'; }

// flag bit 11: valid UTF-8 with at least one non-ASCII character
bool utf8_flag(const uint8_t *s, uint32_t n) {
    bool wide = false;
    for (uint32_t i = 0; i < n;) {
        const uint8_t c = s[i];
        if (c < 0x80) { i++; continue; }
        wide = true;
        uint32_t k, cp;
        if ((c & 0xE0) == 0xC0) { k = 1; cp = c & 0x1F; }
        else if ((c & 0xF0) == 0xE0) { k = 2; cp = c & 0x0F; }
        else if ((c & 0xF8) == 0xF0) { k = 3; cp = c & 0x07; }
        else return false;
        for (uint32_t j = 1; j <= k; j++) {
            if (i + j >= n || (s[i + j] & 0xC0) != 0x80) return false;
            cp = cp << 6 | (s[i + j] & 0x3F);
        }
        if ((k == 1 && cp < 0x80) || (k == 2 && cp < 0x800) || (k == 3 && cp < 0x10000) || cp > 0x10FFFF ||
            (cp >= 0xD800 && cp <= 0xDFFF))
            return false;
        i += k + 1;
    }
    return wide;
}

// MS-DOS date and time of a UTC time, clamped to 1980-01-01 00:00:00 .. 2107-12-31 23:59:58
void dos_time(int64_t t, uint16_t *date, uint16_t *tim) {
    const int64_t lo = 315532800, hi = 4354819198;   // 1980-01-01, 2107-12-31 23:59:58
    time_t c = (time_t)std::min(std::max(t, lo), hi);
    struct tm u;
    gmtime_r(&c, &u);
    *date = (uint16_t)(u.tm_mday + ((u.tm_mon + 1) << 5) + ((u.tm_year + 1900 - 1980) << 9));
    *tim = (uint16_t)(u.tm_sec / 2 + (u.tm_min << 5) + (u.tm_hour << 11));
}

bool has_ext_time(const pbsgpu_zip_entry *e) { return e->mtime >= 0 && e->mtime < (int64_t)1 << 32; }
uint16_t flags_of(const pbsgpu_zip_entry *e) {
    return (uint16_t)((is_dir(e) ? 0 : 0x8) | (utf8_flag(e->name, e->name_len) ? 0x800 : 0));
}
void ext_time(Put &w, const pbsgpu_zip_entry *e) {
    if (!has_ext_time(e)) return;
    w.u16(0x5455); w.u16(5); w.u8(1); w.u32((uint32_t)e->mtime);
}
}  // namespace

extern "C" uint64_t pbsgpu_zip_local_header(const pbsgpu_zip_entry *e, uint8_t *out, uint64_t cap) {
    if (!e || (e->name_len && !e->name)) return 0;
    const uint64_t need = 30 + e->name_len + (has_ext_time(e) ? 9 : 0);
    Put w{out, 0, out && cap >= need};
    uint16_t date, tim;
    dos_time(e->mtime, &date, &tim);
    const bool dir = is_dir(e);
    w.u32(0x04034b50); w.u16(VERSION_20); w.u16(flags_of(e)); w.u16(dir ? 0 : e->method);
    w.u16(tim); w.u16(date);
    w.u32(0); w.u32(0); w.u32(0);   // CRC and sizes: in the data descriptor, or 0 for a directory
    w.u16(e->name_len); w.u16(has_ext_time(e) ? 9 : 0);
    w.bytes(e->name, e->name_len);
    ext_time(w, e);
    return need;
}

extern "C" uint64_t pbsgpu_zip_data_descriptor(const pbsgpu_zip_entry *e, uint8_t *out, uint64_t cap) {
    if (!e || is_dir(e)) return 0;
    const bool z64 = e->comp_size >= U32MAX || e->size >= U32MAX;
    const uint64_t need = z64 ? 24 : 16;
    Put w{out, 0, out && cap >= need};
    w.u32(0x08074b50); w.u32(e->crc);
    if (z64) { w.u64(e->comp_size); w.u64(e->size); }
    else { w.u32((uint32_t)e->comp_size); w.u32((uint32_t)e->size); }
    return need;
}

extern "C" uint64_t pbsgpu_zip_directory(const pbsgpu_zip_entry *e, uint64_t n, uint64_t offset, uint8_t *out, uint64_t cap) {
    if (n && !e) return 0;
    uint64_t need = 0;
    for (int pass = 0; pass < 2; pass++) {   // the size, then (when it fits) the bytes
        Put w{out, 0, pass == 1};
        for (uint64_t k = 0; k < n; k++) {
            const pbsgpu_zip_entry *f = e + k;
            const bool dir = is_dir(f);
            const uint64_t csz = dir ? 0 : f->comp_size, usz = dir ? 0 : f->size;
            const bool zs = usz >= U32MAX, zc = csz >= U32MAX, zo = f->offset >= U32MAX;
            const uint32_t z64 = 8 * (zs + zc + zo);
            const uint32_t extra = (z64 ? 4 + z64 : 0) + (has_ext_time(f) ? 9 : 0);
            uint16_t date, tim;
            dos_time(f->mtime, &date, &tim);
            w.u32(0x02014b50); w.u16(CREATOR_UNIX | VERSION_20); w.u16(z64 ? VERSION_45 : VERSION_20);
            w.u16(flags_of(f)); w.u16(dir ? 0 : f->method); w.u16(tim); w.u16(date);
            w.u32(dir ? 0 : f->crc);
            w.u32(zc ? U32MAX : (uint32_t)csz); w.u32(zs ? U32MAX : (uint32_t)usz);
            w.u16(f->name_len); w.u16(extra); w.u16(0);   // comment
            w.u16(0); w.u16(0);                            // disk, internal attributes
            w.u32(f->mode << 16 | (dir ? 0x10 : 0));
            w.u32(zo ? U32MAX : (uint32_t)f->offset);
            w.bytes(f->name, f->name_len);
            if (z64) {   // APPNOTE 4.5.3: only the fields that overflow, in this order
                w.u16(0x0001); w.u16(z64);
                if (zs) w.u64(usz);
                if (zc) w.u64(csz);
                if (zo) w.u64(f->offset);
            }
            ext_time(w, f);
        }
        const uint64_t size = w.q, end = offset + size;
        if (n >= 0xFFFF || size >= U32MAX || offset >= U32MAX) {
            w.u32(0x06064b50); w.u64(44); w.u16(CREATOR_UNIX | VERSION_45); w.u16(VERSION_45);
            w.u32(0); w.u32(0); w.u64(n); w.u64(n); w.u64(size); w.u64(offset);
            w.u32(0x07064b50); w.u32(0); w.u64(end); w.u32(1);
        }
        w.u32(0x06054b50); w.u16(0); w.u16(0);
        w.u16((uint32_t)std::min<uint64_t>(n, 0xFFFF)); w.u16((uint32_t)std::min<uint64_t>(n, 0xFFFF));
        w.u32((uint32_t)std::min<uint64_t>(size, U32MAX)); w.u32((uint32_t)std::min<uint64_t>(offset, U32MAX));
        w.u16(0);
        need = w.q;
        if (!out || cap < need) break;
    }
    return need;
}
