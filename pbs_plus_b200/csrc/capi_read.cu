// pbs_plus_b200/csrc/capi_read.cu -- C ABI of the archive reader (f3, read side): byte ranges of the archive an index
// describes, served from a cache of verified chunks in device memory.
// The index (end offsets, digests, chunk lengths) and the cache's bookkeeping live on the host; the device holds only
// the cache.  Blobs are decoded and verified by pbsgpu_blob_decode (K6, K11, K13, K3) straight into their cache slots,
// and K14 copies the pieces of the ranges out of the cache.
#include <algorithm>
#include <cstring>
#include <deque>
#include <unordered_map>

#include "host.hpp"

using namespace pbsgpu;

static constexpr uint64_t READER_DEFAULT_CACHE = 256ull << 20;   // pxar-mount's --cache-size default
static constexpr uint64_t READER_STAGE_MAX = 256ull << 20;       // staging of a host `out`
static constexpr uint32_t READER_PIECE_BATCH = 1u << 20;         // pieces per K14 launch
static const uint8_t PXAR_PAYLOAD_LE[8] = {0x25, 0x1a, 0x7c, 0x0b, 0x1b, 0x7a, 0x14, 0x28};   // 0x28147A1B0B7C1A25

struct pbsgpu_reader {
    pbsgpu_ctx *ctx;
    const pbsgpu_crypt *crypt;
    std::vector<uint64_t> ends, clen;   // per chunk: end offset in the archive, length
    std::vector<uint8_t> digests;       // per chunk: 32 bytes
    uint8_t *cache = nullptr;
    // The ring: slots in insertion order from the oldest.  They lie at ascending offsets from the oldest one up, then
    // (after a wrap) from 0 up to the cursor, so the slots a new one overwrites are always a prefix of `ring`.  A slot
    // stays in the ring after its chunk failed or was dropped; `held` names the slots of verified chunks.
    struct Slot { uint64_t chunk, off, bytes, seq, gen; };
    struct Held { uint64_t off, seq; };
    uint64_t cap = 0, cursor = 0, seq = 0, gen = 0;
    std::deque<Slot> ring;
    std::unordered_map<uint64_t, Held> held;
    bool image = false;   // over a fixed index: no pxar headers, PBSGPU_READ_PAYLOAD is refused
    // sparse calls: the digests of clen zero bytes for the (at most two) chunk lengths of an image, or for the longest
    // chunk of a .didx reader, computed on first use
    bool zero_known = false;
    uint64_t zero_len[2] = {0, 0};
    uint8_t zero_dig[2][32];
};

static uint64_t slot_bytes(uint64_t len) { return std::max<uint64_t>(256, (len + 255) & ~255ull); }

// where a new slot of `bytes` goes: at the cursor, or at 0 when it would run past the ring's end
static uint64_t slot_at(const pbsgpu_reader *r, uint64_t bytes) { return r->cursor + bytes <= r->cap ? r->cursor : 0; }
// does a new slot of `bytes` at `at` overwrite s?  On a wrap, also every slot between the cursor and the end.
static bool overwrites(const pbsgpu_reader *r, const pbsgpu_reader::Slot &s, uint64_t at, uint64_t bytes) {
    return at == r->cursor ? s.off >= at && s.off < at + bytes : s.off >= r->cursor || s.off < bytes;
}
static bool overwrites_gen(const pbsgpu_reader *r, uint64_t bytes, uint64_t gen) {
    const uint64_t at = slot_at(r, bytes);
    for (const auto &s : r->ring) {
        if (!overwrites(r, s, at, bytes)) return false;
        if (s.gen == gen) return true;
    }
    return false;
}
static const pbsgpu_reader::Slot &place(pbsgpu_reader *r, uint64_t chunk, uint64_t bytes, uint64_t gen) {
    const uint64_t at = slot_at(r, bytes);
    while (!r->ring.empty() && overwrites(r, r->ring.front(), at, bytes)) {
        const auto &s = r->ring.front();
        auto h = r->held.find(s.chunk);
        if (h != r->held.end() && h->second.seq == s.seq) r->held.erase(h);
        r->ring.pop_front();
    }
    r->cursor = at + bytes;
    r->ring.push_back({chunk, at, bytes, ++r->seq, gen});
    return r->ring.back();
}

// The chunk lengths from r->ends, then the cache; frees r on failure.
static int reader_start(pbsgpu_reader *r, uint64_t cache_bytes, pbsgpu_reader **out) {
    pbsgpu_ctx *ctx = r->ctx;
    const uint64_t n = r->ends.size();
    r->clen.resize(n);
    uint64_t largest = 0;
    for (uint64_t c = 0; c < n; c++) {
        r->clen[c] = r->ends[c] - (c ? r->ends[c - 1] : 0);
        if (r->clen[c] >= (1ull << 32)) { delete r; return fail(ctx, PBSGPU_EINVAL, "index chunk %llu: 2^32 bytes or more", (unsigned long long)c); }
        largest = std::max(largest, slot_bytes(r->clen[c]));
    }
    r->cap = std::max<uint64_t>((cache_bytes ? cache_bytes : READER_DEFAULT_CACHE) & ~255ull, largest);
    // 16 bytes of slack: K14's word path reads up to 3 bytes past a piece's last byte
    if (cudaMalloc((void **)&r->cache, r->cap + 16) != cudaSuccess) {
        (void)cudaGetLastError();
        delete r;
        return fail(ctx, PBSGPU_ENOMEM, "reader cache of %llu bytes failed", (unsigned long long)(cache_bytes ? cache_bytes : READER_DEFAULT_CACHE));
    }
    *out = r;
    return PBSGPU_OK;
}

extern "C" int pbsgpu_reader_open(pbsgpu_ctx *ctx, const uint8_t *didx, uint64_t size, const pbsgpu_crypt *crypt,
                                  uint64_t cache_bytes, pbsgpu_reader **out) {
    if (!ctx || !didx || !out || (crypt && crypt->ctx != ctx)) return PBSGPU_EINVAL;
    Guard g(ctx);
    uint64_t n = 0;
    if (int rc = pbsgpu_didx_parse(ctx, didx, size, nullptr, nullptr, 0, &n, 0)) return rc;
    pbsgpu_reader *r = new pbsgpu_reader{};
    r->ctx = ctx; r->crypt = crypt;
    r->ends.resize(n); r->digests.resize(n * 32);
    if (int rc = pbsgpu_didx_parse(ctx, didx, size, r->ends.data(), r->digests.data(), n, &n, 1)) { delete r; return rc; }
    return reader_start(r, cache_bytes, out);
}

// The same reader over a fixed index: the end offsets are synthesized, so lookup, cache, decode and gather are shared.
extern "C" int pbsgpu_reader_open_fidx(pbsgpu_ctx *ctx, const uint8_t *fidx, uint64_t bytes, const pbsgpu_crypt *crypt,
                                       uint64_t cache_bytes, pbsgpu_reader **out) {
    if (!ctx || !fidx || !out || (crypt && crypt->ctx != ctx)) return PBSGPU_EINVAL;
    Guard g(ctx);
    uint64_t n = 0, size = 0, cs = 0;
    if (int rc = pbsgpu_fidx_parse(ctx, fidx, bytes, &size, &cs, nullptr, 0, &n, 0)) return rc;
    pbsgpu_reader *r = new pbsgpu_reader{};
    r->ctx = ctx; r->crypt = crypt; r->image = true;
    r->digests.resize(n * 32);
    if (int rc = pbsgpu_fidx_parse(ctx, fidx, bytes, nullptr, nullptr, r->digests.data(), n, &n, 1)) { delete r; return rc; }
    r->ends.resize(n);
    for (uint64_t c = 0; c < n; c++) r->ends[c] = std::min((c + 1) * cs, size);
    return reader_start(r, cache_bytes, out);
}

extern "C" void pbsgpu_reader_close(pbsgpu_reader *r) {
    if (!r) return;
    {
        Guard g(r->ctx);
        if (r->crypt && (cudaMemset(r->cache, 0, r->cap + 16) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess))
            (void)cudaGetLastError();
        cudaFree(r->cache);
    }
    delete r;
}

extern "C" uint64_t pbsgpu_reader_size(const pbsgpu_reader *r) { return r && !r->ends.empty() ? r->ends.back() : 0; }

// The pieces of the archive bytes [lo, hi): fn(chunk, offset in the chunk, length, offset from lo), in chunk order;
// chunks of length 0 are skipped.
template <typename F> static void for_pieces(const pbsgpu_reader *r, uint64_t lo, uint64_t hi, F fn) {
    if (lo >= hi) return;
    uint64_t c = std::upper_bound(r->ends.begin(), r->ends.end(), lo) - r->ends.begin();
    for (; c < r->ends.size(); c++) {
        const uint64_t start = r->ends[c] - r->clen[c];
        if (start >= hi) break;
        if (r->clen[c] == 0) continue;
        const uint64_t a = std::max(lo, start), e = std::min(hi, r->ends[c]);
        fn(c, a - start, e - a, a - lo);
    }
}

// The digests of clen zero bytes, plain or keyed with the reader's crypt as the index's digests are: K3 through the
// SHA-256 batch calls, once per reader.  An image: its two chunk lengths (chunk_size and the last chunk's).  A .didx
// reader: its longest chunk length, the one that carries zero runs (a zero window hashes to 0, so a zero run is only
// cut at the chunker's maximum) -- but only when two or more chunks of that length share a digest.  That digest is one
// serial SHA-256 chain over the longest length (16 MiB at a 4 MiB average), which costs more than fetching and decoding
// one chunk, so a digest the index holds once is not worth identifying; without a repeat zero_len[0] stays 0 and no
// chunk is served by digest (for_pieces never visits a chunk of length 0).
static bool longest_digest_repeats(const pbsgpu_reader *r, uint64_t longest) {
    std::vector<const uint8_t *> d;
    for (uint64_t c = 0; c < r->clen.size(); c++)
        if (r->clen[c] == longest) d.push_back(r->digests.data() + 32 * c);
    std::sort(d.begin(), d.end(), [](const uint8_t *a, const uint8_t *b) { return memcmp(a, b, 32) < 0; });
    for (size_t k = 1; k < d.size(); k++)
        if (memcmp(d[k - 1], d[k], 32) == 0) return true;
    return false;
}
static int zero_digests(pbsgpu_reader *r) {
    if (r->zero_known || r->ends.empty()) return PBSGPU_OK;
    if (!r->image) {
        const uint64_t longest = *std::max_element(r->clen.begin(), r->clen.end());
        if (!longest_digest_repeats(r, longest)) {
            r->zero_known = true;
            return PBSGPU_OK;
        }
    }
    // an image's longest is its first: every chunk but the last is chunk_size
    r->zero_len[0] = r->image ? r->clen.front() : *std::max_element(r->clen.begin(), r->clen.end());
    r->zero_len[1] = r->image ? r->clen.back() : 0;
    const uint32_t k = r->image ? 2 : 1;
    const std::vector<uint8_t> zeros(r->zero_len[0]);
    const uint64_t at[2] = {0, 0};
    if (int rc = r->crypt ? pbsgpu_sha256_keyed_batch(r->ctx, r->crypt, zeros.data(), at, r->zero_len, k, r->zero_dig[0])
                          : pbsgpu_sha256_batch(r->ctx, zeros.data(), at, r->zero_len, k, r->zero_dig[0]))
        return rc;
    r->zero_known = true;
    return PBSGPU_OK;
}
// chunk c is served by its digest in a sparse call (after zero_digests): a zero chunk -- its index digest is the digest
// of clen[c] zero bytes -- whose start and end lie on 4 KiB block boundaries (the end may be the image's end), so no
// block part holds both its zeros and another chunk's bytes.  A zero chunk that cuts a block (a chunk size that is not
// a multiple of 4096) is read like a data chunk: skipping it would split that block's data between two runs.
static bool zero_chunk(const pbsgpu_reader *r, uint64_t c) {
    const uint64_t start = r->ends[c] - r->clen[c];
    if (start % ZERO_BLOCK || (r->ends[c] % ZERO_BLOCK && r->ends[c] != r->ends.back())) return false;
    const int k = r->clen[c] == r->zero_len[0] ? 0 : r->clen[c] == r->zero_len[1] ? 1 : -1;
    return k >= 0 && memcmp(r->digests.data() + 32 * c, r->zero_dig[k], 32) == 0;
}
// chunk c of a .didx reader is served by its digest in a file-sparse call (after zero_digests): a zero chunk of the
// index's longest length, when that length holds a repeated digest.  Its bounds need not be block boundaries: the call stages the zeros of the blocks it shares
// with data chunks itself.
static bool file_zero_chunk(const pbsgpu_reader *r, uint64_t c) {
    return r->clen[c] == r->zero_len[0] && memcmp(r->digests.data() + 32 * c, r->zero_dig[0], 32) == 0;
}

// The arguments every call checks: flags, and every range (with its PAYLOAD header) inside the archive.
static int check_ranges(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags) {
    if (flags & ~PBSGPU_READ_PAYLOAD) return fail(r->ctx, PBSGPU_EINVAL, "unknown read flags 0x%x", flags);
    if (r->image && (flags & PBSGPU_READ_PAYLOAD)) return fail(r->ctx, PBSGPU_EINVAL, "an image has no pxar PAYLOAD headers");
    const uint64_t hs = flags & PBSGPU_READ_PAYLOAD ? 16 : 0, size = pbsgpu_reader_size(r);
    for (uint32_t i = 0; i < n; i++)
        if (off[i] > size || len[i] > size - off[i] || hs > size - off[i] - len[i])
            return fail(r->ctx, PBSGPU_EINVAL, "range %u ends past the archive (%llu bytes)", i, (unsigned long long)size);
    return PBSGPU_OK;
}
// The file-sparse form: a .didx reader, every file (header and content) inside the archive, every range inside its file.
static int check_file_ranges(pbsgpu_reader *r, const uint64_t *file_off, const uint64_t *file_size, const uint64_t *pos,
                             const uint64_t *len, uint32_t n) {
    if (r->image) return fail(r->ctx, PBSGPU_EINVAL, "file sparse: an image has no pxar files");
    const uint64_t size = pbsgpu_reader_size(r);
    for (uint32_t i = 0; i < n; i++) {
        if (file_off[i] > size || 16 > size - file_off[i] || file_size[i] > size - file_off[i] - 16)
            return fail(r->ctx, PBSGPU_EINVAL, "range %u: its file ends past the archive (%llu bytes)", i, (unsigned long long)size);
        if (pos[i] > file_size[i] || len[i] > file_size[i] - pos[i])
            return fail(r->ctx, PBSGPU_EINVAL, "range %u: [pos, pos + len) is not inside its file", i);
    }
    return PBSGPU_OK;
}
// Does the 16-byte PAYLOAD header h announce `size` content bytes?
static bool payload_header_ok(const uint8_t *h, uint64_t size) {
    uint8_t want[16];
    memcpy(want, PXAR_PAYLOAD_LE, 8);
    for (int k = 0; k < 8; k++) want[8 + k] = (uint8_t)((16 + size) >> (8 * k));
    return memcmp(h, want, 16) == 0;
}

// The plans' common tail: the needed chunks ascending and without repeats, with their digests.
static int plan_out(pbsgpu_reader *r, std::vector<uint64_t> &need, uint64_t *chunk, uint8_t *digest, uint64_t cap,
                    uint64_t *n_out) {
    std::sort(need.begin(), need.end());
    need.erase(std::unique(need.begin(), need.end()), need.end());
    *n_out = need.size();
    if (need.size() > cap) return fail(r->ctx, PBSGPU_ERANGE, "plan capacity %llu < %llu chunks", (unsigned long long)cap, (unsigned long long)need.size());
    for (size_t k = 0; k < need.size(); k++) {
        chunk[k] = need[k];
        if (digest) memcpy(digest + 32 * k, r->digests.data() + 32 * need[k], 32);
    }
    return PBSGPU_OK;
}

extern "C" int pbsgpu_reader_plan(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                                  uint64_t *chunk, uint8_t *digest, uint64_t cap, uint64_t *n_out) {
    if (!r || !n_out || (n && (!off || !len)) || (cap && !chunk)) return PBSGPU_EINVAL;
    Guard g(r->ctx);
    const bool sparse = flags & PBSGPU_READ_SPARSE;   // plan's flag alone: check_ranges refuses it for the reads
    flags &= ~PBSGPU_READ_SPARSE;
    if (sparse && !r->image) return fail(r->ctx, PBSGPU_EINVAL, "PBSGPU_READ_SPARSE needs a .fidx reader");
    if (int rc = check_ranges(r, off, len, n, flags)) return rc;
    if (sparse)
        if (int rc = zero_digests(r)) return rc;
    const uint64_t hs = flags & PBSGPU_READ_PAYLOAD ? 16 : 0;
    std::vector<uint64_t> need;
    for (uint32_t i = 0; i < n; i++)
        for_pieces(r, off[i], off[i] + hs + len[i], [&](uint64_t c, uint64_t, uint64_t, uint64_t) {
            if (!r->held.count(c) && !(sparse && zero_chunk(r, c))) need.push_back(c);
        });
    return plan_out(r, need, chunk, digest, cap, n_out);
}

extern "C" int pbsgpu_reader_plan_file_sparse(pbsgpu_reader *r, const uint64_t *file_off, const uint64_t *file_size,
                                              const uint64_t *pos, const uint64_t *len, uint32_t n, uint64_t *chunk,
                                              uint8_t *digest, uint64_t cap, uint64_t *n_out) {
    if (!r || !n_out || (n && (!file_off || !file_size || !pos || !len)) || (cap && !chunk)) return PBSGPU_EINVAL;
    Guard g(r->ctx);
    if (int rc = check_file_ranges(r, file_off, file_size, pos, len, n)) return rc;
    if (int rc = zero_digests(r)) return rc;
    std::vector<uint64_t> need;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t a = file_off[i] + 16 + pos[i];   // a range at pos 0 also reads its file's header
        for_pieces(r, pos[i] ? a : file_off[i], a + len[i], [&](uint64_t c, uint64_t, uint64_t, uint64_t) {
            if (!r->held.count(c) && !file_zero_chunk(r, c)) need.push_back(c);
        });
    }
    return plan_out(r, need, chunk, digest, cap, n_out);
}

namespace {
// One (range, chunk) intersection: `len` bytes at `coff` in the chunk go to `dst` -- an offset into `out` (content) or
// into the header scratch (hdr, PAYLOAD headers).  cached: the chunk was held when the call started.
struct RawPiece { uint64_t chunk, coff, len, dst; uint32_t range; bool hdr, cached; };

// K14 launches of pieces from the cache: to the header scratch, to a device `out`, or through a bounded staging buffer
// to a host `out` (one D2H copy per run of pieces contiguous both in the staging buffer and in `out`).
struct Gather {
    Blocking &b;
    pbsgpu_reader *r;
    uint8_t *out, *d_hdr, *stage = nullptr;
    bool out_dev;
    uint64_t stage_cap = 0, stage_used = 0;
    ReadPiece *d_pieces = nullptr;
    uint64_t *d_first = nullptr;
    std::vector<ReadPiece> pieces;
    std::vector<uint64_t> first;
    struct Run { uint64_t stage, out, len; };
    std::vector<Run> runs;

    int flush() {
        const uint32_t np = (uint32_t)pieces.size();
        if (np) {
            first.assign(np + 1, 0);
            for (uint32_t p = 0; p < np; p++) first[p + 1] = first[p] + (pieces[p].len + READ_TILE - 1) / READ_TILE;
            if (b.ok()) b.e = cudaMemcpyAsync(d_pieces, pieces.data(), np * sizeof(ReadPiece), cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(d_first, first.data(), (np + 1) * 8ull, cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = launch_read_gather(d_pieces, d_first, np, first[np], r->ctx->sm_count, b.st);
        }
        for (const Run &u : runs)
            if (b.ok()) b.e = cudaMemcpyAsync(out + u.out, stage + u.stage, u.len, cudaMemcpyDeviceToHost, b.st);
        pieces.clear(); runs.clear(); stage_used = 0;
        return b.finish("reader gather");
    }
    int add(const RawPiece &q, const uint8_t *src) {   // src: the chunk's cache slot (or the stage q.coff is into)
        uint64_t done = 0;
        while (done < q.len) {
            if (pieces.size() == READER_PIECE_BATCH || (!q.hdr && !out_dev && stage_used == stage_cap))
                if (int rc = flush()) return rc;
            uint64_t take = q.len - done, dst;
            if (q.hdr) dst = (uint64_t)(uintptr_t)d_hdr + q.dst + done;
            else if (out_dev) dst = (uint64_t)(uintptr_t)out + q.dst + done;
            else {
                take = std::min(take, stage_cap - stage_used);
                dst = (uint64_t)(uintptr_t)stage + stage_used;
                if (!runs.empty() && runs.back().stage + runs.back().len == stage_used && runs.back().out + runs.back().len == q.dst + done)
                    runs.back().len += take;
                else
                    runs.push_back({stage_used, q.dst + done, take});
                stage_used += take;
            }
            pieces.push_back({(uint64_t)(uintptr_t)src + q.coff + done, dst, take});
            done += take;
        }
        return PBSGPU_OK;
    }
};
}  // namespace

extern "C" int pbsgpu_reader_read(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                                  const void *blob_base, const uint64_t *blob_off, const uint64_t *blob_len,
                                  const uint64_t *blob_chunk, uint32_t n_blobs,
                                  uint8_t *out, const uint64_t *out_off, int32_t *status, int32_t *blob_status) {
    if (!r || (n && (!off || !len || !out || !out_off || !status)) ||
        (n_blobs && (!blob_base || !blob_off || !blob_len || !blob_chunk)))
        return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = r->ctx;
    Guard g(ctx);
    if (int rc = check_ranges(r, off, len, n, flags)) return rc;
    const uint64_t hs = flags & PBSGPU_READ_PAYLOAD ? 16 : 0, m = r->ends.size();
    std::unordered_map<uint64_t, uint32_t> given;   // chunk -> its blob
    for (uint32_t j = 0; j < n_blobs; j++) {
        if (blob_chunk[j] >= m) return fail(ctx, PBSGPU_EINVAL, "blob %u: chunk %llu not in the index", j, (unsigned long long)blob_chunk[j]);
        if (!given.emplace(blob_chunk[j], j).second) return fail(ctx, PBSGPU_EINVAL, "blob %u: chunk %llu given twice", j, (unsigned long long)blob_chunk[j]);
        if (blob_off[j] + blob_len[j] < blob_off[j]) return fail(ctx, PBSGPU_EINVAL, "blob %u: range wraps around", j);
    }
    // 1. the given chunks leave the cache
    for (uint32_t j = 0; j < n_blobs; j++) r->held.erase(blob_chunk[j]);
    // the pieces, range by range in chunk order
    std::vector<RawPiece> raw;
    uint64_t host_bytes = 0;
    for (uint32_t i = 0; i < n; i++) {
        for_pieces(r, off[i], off[i] + hs + len[i], [&](uint64_t c, uint64_t coff, uint64_t l, uint64_t at) {
            const bool cached = r->held.count(c) != 0;
            if (at < hs) {   // the part of the PAYLOAD header in this chunk
                const uint64_t hl = std::min(l, hs - at);
                raw.push_back({c, coff, hl, 16ull * i + at, i, true, cached});
                coff += hl; l -= hl; at += hl;
            }
            if (l) raw.push_back({c, coff, l, out_off[i] + at - hs, i, false, cached});
        });
    }
    const bool out_dev = out && pbsgpu_is_device_ptr(out);
    for (const RawPiece &q : raw) if (!q.hdr) host_bytes += q.len;
    Blocking b(ctx, ctx->streams[0]);
    Gather ga{b, r, out, nullptr};
    ga.out_dev = out_dev;
    const uint32_t pcap = (uint32_t)std::min<uint64_t>(raw.size() + 1, READER_PIECE_BATCH) * 2;   // a split piece adds one
    ga.d_pieces = b.get<ReadPiece>(pcap);
    ga.d_first = b.get<uint64_t>(pcap + 1);
    ga.pieces.reserve(pcap);
    if (hs && n) ga.d_hdr = b.get<uint8_t>(16ull * n + 16);
    if (!out_dev && host_bytes) {
        ga.stage_cap = std::min(host_bytes, READER_STAGE_MAX);
        ga.stage = b.get<uint8_t>(ga.stage_cap);
    }
    if (!ga.d_pieces || !ga.d_first || (hs && n && !ga.d_hdr) || (!out_dev && host_bytes && !ga.stage))
        return fail(ctx, PBSGPU_ENOMEM, "reader gather buffers failed");
    // 2. the pieces of chunks that were cached, before any decode can overwrite them
    for (const RawPiece &q : raw)
        if (q.cached)
            if (int rc = ga.add(q, r->cache + r->held[q.chunk].off)) return rc;
    if (int rc = ga.flush()) return rc;
    // 3. the blobs, in groups whose slots do not overwrite each other; each group's pieces are copied right after it
    std::vector<int32_t> bst(n_blobs, PBSGPU_DEC_OK);
    std::vector<uint64_t> slot(n_blobs), slot_seq(n_blobs), by_chunk(raw.size());
    for (size_t k = 0; k < raw.size(); k++) by_chunk[k] = k;
    std::stable_sort(by_chunk.begin(), by_chunk.end(), [&](uint64_t x, uint64_t y) { return raw[x].chunk < raw[y].chunk; });
    std::vector<uint64_t> go, gl, gcl, gout, mine;
    std::vector<uint8_t> gdig;
    auto run_group = [&](uint32_t j0, uint32_t j1) -> int {
        if (j0 == j1) return PBSGPU_OK;
        uint64_t lo = ~0ull;
        for (uint32_t j = j0; j < j1; j++) lo = std::min(lo, blob_off[j]);
        go.clear(); gl.clear(); gcl.clear(); gout.clear(); gdig.clear();
        for (uint32_t j = j0; j < j1; j++) {
            const uint64_t c = blob_chunk[j];
            go.push_back(blob_off[j] - lo); gl.push_back(blob_len[j]); gcl.push_back(r->clen[c]); gout.push_back(slot[j]);
            gdig.insert(gdig.end(), r->digests.begin() + 32 * c, r->digests.begin() + 32 * c + 32);
        }
        // host blobs are staged from `lo` on, so a group copies only its own span
        if (int rc = pbsgpu_blob_decode(ctx, r->crypt, (const uint8_t *)blob_base + lo, go.data(), gl.data(), j1 - j0, gcl.data(),
                                        gdig.data(), r->cache, gout.data(), bst.data() + j0, nullptr))
            return rc;
        mine.clear();
        for (uint32_t j = j0; j < j1; j++) {
            if (bst[j] != PBSGPU_DEC_OK) continue;
            const uint64_t c = blob_chunk[j];
            r->held[c] = {slot[j], slot_seq[j]};
            auto lo_it = std::lower_bound(by_chunk.begin(), by_chunk.end(), c, [&](uint64_t k, uint64_t v) { return raw[k].chunk < v; });
            for (; lo_it != by_chunk.end() && raw[*lo_it].chunk == c; ++lo_it) mine.push_back(*lo_it);
        }
        std::sort(mine.begin(), mine.end());   // range order: runs of a host `out` coalesce
        for (uint64_t k : mine)
            if (int rc = ga.add(raw[k], r->cache + slot[given[raw[k].chunk]])) return rc;
        return ga.flush();
    };
    uint32_t j0 = 0;
    uint64_t gen = ++r->gen;
    for (uint32_t j = 0; j < n_blobs; j++) {
        const uint64_t bytes = slot_bytes(r->clen[blob_chunk[j]]);
        if (overwrites_gen(r, bytes, gen)) {
            if (int rc = run_group(j0, j)) return rc;
            j0 = j;
            gen = ++r->gen;
        }
        const auto &s = place(r, blob_chunk[j], bytes, gen);
        slot[j] = s.off; slot_seq[j] = s.seq;
    }
    if (int rc = run_group(j0, n_blobs)) return rc;
    if (blob_status) memcpy(blob_status, bst.data(), n_blobs * sizeof(int32_t));
    // 4. statuses: the first failing chunk of each range in chunk order, then its PAYLOAD header
    for (uint32_t i = 0; i < n; i++) status[i] = PBSGPU_DEC_OK;
    for (const RawPiece &q : raw) {
        if (status[q.range] != PBSGPU_DEC_OK) continue;
        auto it = given.find(q.chunk);
        if (it != given.end()) status[q.range] = bst[it->second];
        else if (!q.cached) status[q.range] = PBSGPU_DEC_MISSING;
    }
    if (hs && n) {
        std::vector<uint8_t> hdr(16ull * n);
        if (b.ok()) b.e = cudaMemcpyAsync(hdr.data(), ga.d_hdr, hdr.size(), cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("reader headers")) return rc;
        for (uint32_t i = 0; i < n; i++)
            if (status[i] == PBSGPU_DEC_OK && !payload_header_ok(hdr.data() + 16ull * i, len[i])) status[i] = PBSGPU_DEC_BAD_HEADER;
    }
    return PBSGPU_OK;
}

// The zip restore's read: the ranges go through pbsgpu_reader_read into a device stage owned by this call, and only the
// ranges whose status is OK are deflated from there (pbsgpu_deflate_batch, or pbsgpu_deflate_batch_lzc with
// PBSGPU_READ_DEFLATE_LZC) into the caller's host memory, so file bytes cross PCIe compressed and no byte of a failed
// range reaches `out`.
extern "C" int pbsgpu_reader_read_deflate(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                                          const uint8_t *more, const void *blob_base, const uint64_t *blob_off,
                                          const uint64_t *blob_len, const uint64_t *blob_chunk, uint32_t n_blobs, uint8_t *out,
                                          const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out, int32_t *status,
                                          int32_t *blob_status) {
    if (!r || (n && (!off || !len || !out || !out_off || !out_len || !status)) ||
        (n_blobs && (!blob_base || !blob_off || !blob_len || !blob_chunk)))
        return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = r->ctx;
    Guard g(ctx);
    const bool lzc = flags & PBSGPU_READ_DEFLATE_LZC;   // this call's flag alone: the read below never sees it
    flags &= ~PBSGPU_READ_DEFLATE_LZC;
    if (n && pbsgpu_is_device_ptr(out)) return fail(ctx, PBSGPU_EINVAL, "read_deflate: out must be host memory");
    for (uint32_t i = 0; i < n; i++)
        if (more && more[i] && len[i] % DEFLATE_SEGMENT)
            return fail(ctx, PBSGPU_EINVAL, "range %u: a piece that a later call continues must be a multiple of 128 KiB", i);
    if (int rc = check_ranges(r, off, len, n, flags)) return rc;
    std::vector<uint64_t> soff(n);
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) { soff[i] = total; total += len[i]; }
    Blocking b(ctx, ctx->streams[0]);
    uint8_t *stage = b.get<uint8_t>(total + 16);
    if (!stage) return fail(ctx, PBSGPU_ENOMEM, "read_deflate: device stage of %llu bytes failed", (unsigned long long)total);
    if (int rc = pbsgpu_reader_read(r, off, len, n, flags, blob_base, blob_off, blob_len, blob_chunk, n_blobs, stage,
                                    soff.data(), status, blob_status))
        return rc;
    std::vector<uint64_t> ko, kl, koo, klen;
    std::vector<uint8_t> km;
    std::vector<uint32_t> idx, kcrc;
    for (uint32_t i = 0; i < n; i++) {
        out_len[i] = 0;
        if (crc_out) crc_out[i] = 0;
        if (status[i] != PBSGPU_DEC_OK) continue;
        idx.push_back(i); ko.push_back(soff[i]); kl.push_back(len[i]); koo.push_back(out_off[i]);
        km.push_back(more && more[i]);
    }
    const uint32_t k = (uint32_t)idx.size();
    if (k == 0) return PBSGPU_OK;
    klen.resize(k); kcrc.resize(k);
    if (int rc = (lzc ? pbsgpu_deflate_batch_lzc : pbsgpu_deflate_batch)(ctx, stage, ko.data(), kl.data(), k, km.data(), out,
                                                                         koo.data(), klen.data(), crc_out ? kcrc.data() : nullptr))
        return rc;
    for (uint32_t j = 0; j < k; j++) {
        out_len[idx[j]] = klen[j];
        if (crc_out) crc_out[idx[j]] = kcrc[j];
    }
    return PBSGPU_OK;
}

namespace {
// A staged run of a sparse read: `len` bytes of range `range` at block coordinate `off` (an image offset, or an offset
// into a file's content) that lie at `soff` in the call's device stage, with soff = off mod 16 so K17's vector loads are
// aligned on whole blocks.  Two runs of a range are apart by at least one whole hole block, so no block part spans two.
struct SparseRun { uint64_t off, len, soff; uint32_t range; };
}  // namespace

// The sparse reads' argument checks: out in host memory, and ext_cap at least sum ceil(B_i / 2), with B_i the block
// parts of [at[i], at[i] + len[i]) in block coordinates.  bit0[i]: the bit of range i's first block part.
static int sparse_bits(pbsgpu_reader *r, const uint64_t *at, const uint64_t *len, uint32_t n, const uint8_t *out,
                       uint64_t ext_cap, const char *what, std::vector<uint64_t> &bit0) {
    if (n && pbsgpu_is_device_ptr(out)) return fail(r->ctx, PBSGPU_EINVAL, "%s: out must be host memory", what);
    bit0.assign(n + 1, 0);
    uint64_t bound = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t parts = len[i] ? (at[i] + len[i] - 1) / ZERO_BLOCK - at[i] / ZERO_BLOCK + 1 : 0;
        bit0[i + 1] = bit0[i] + parts;
        bound += (parts + 1) / 2;
    }
    if (ext_cap < bound)
        return fail(r->ctx, PBSGPU_EINVAL, "%s: ext_cap %llu < %llu, the most extents the ranges can have", what,
                    (unsigned long long)ext_cap, (unsigned long long)bound);
    return PBSGPU_OK;
}

// The sparse reads' common tail, once the runs are staged and the statuses known: K17 maps the all-zero block parts of
// the runs of the ranges that are OK, the extents are the maximal runs of the other block parts, and K14 copies their
// bytes to the caller's host memory, packed per range.  A block part no run covers keeps the preset bit: a hole.
static int sparse_extents(pbsgpu_reader *r, Blocking &b, const std::vector<SparseRun> &runs, const uint8_t *dstage,
                          const uint64_t *at, const std::vector<uint64_t> &bit0, uint32_t n, uint8_t *out,
                          const uint64_t *out_off, uint64_t *ext, uint64_t *ext_first, const int32_t *status,
                          const char *what) {
    pbsgpu_ctx *ctx = r->ctx;
    const uint32_t nr = (uint32_t)runs.size();
    std::vector<ZeroRun> zr;
    std::vector<uint64_t> part_first(1, 0);
    for (const SparseRun &u : runs) {
        if (status[u.range] != PBSGPU_DEC_OK) continue;
        const uint64_t b0 = u.off / ZERO_BLOCK, b1 = (u.off + u.len - 1) / ZERO_BLOCK;
        zr.push_back({(uint64_t)(uintptr_t)dstage + u.soff, u.off, u.len, bit0[u.range] + b0 - at[u.range] / ZERO_BLOCK});
        part_first.push_back(part_first.back() + b1 - b0 + 1);
    }
    std::vector<uint32_t> bits;
    if (!zr.empty()) {
        const uint64_t words = (bit0[n] + 31) / 32;
        bits.resize(words);
        uint32_t *d_bits = b.get<uint32_t>(words);
        const ZeroRun *d_runs = b.upload(zr.data(), zr.size());
        const uint64_t *d_first = b.upload(part_first.data(), part_first.size());
        if (!d_bits || !d_runs || !d_first) return fail(ctx, PBSGPU_ENOMEM, "%s: zero map buffers failed", what);
        if (b.ok()) b.e = cudaMemsetAsync(d_bits, 0xff, words * 4, b.st);
        if (b.ok()) b.e = launch_zero_map(d_runs, d_first, (uint32_t)zr.size(), part_first.back(), d_bits, ctx->sm_count, b.st);
        if (b.ok()) b.e = cudaMemcpyAsync(bits.data(), d_bits, words * 4, cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("sparse zero map")) return rc;
    }
    // the extents: an extent lies in one run (SparseRun), so its dstage bytes are contiguous
    std::vector<uint64_t> esrc;   // per extent: its offset in dstage
    uint64_t ne = 0, host_bytes = 0;
    if (n) ext_first[0] = 0;
    for (uint32_t i = 0, k = 0; i < n; i++) {
        const uint64_t e0 = ne;
        for (; k < nr && runs[k].range == i; k++) {
            const SparseRun &u = runs[k];
            if (status[i] != PBSGPU_DEC_OK) continue;
            const uint64_t b0 = u.off / ZERO_BLOCK, b1 = (u.off + u.len - 1) / ZERO_BLOCK;
            for (uint64_t blk = b0; blk <= b1; blk++) {
                const uint64_t bit = bit0[i] + blk - at[i] / ZERO_BLOCK;
                if (bits[bit >> 5] >> (bit & 31) & 1) continue;   // a hole
                const uint64_t lo = std::max(u.off, blk * ZERO_BLOCK), hi = std::min(u.off + u.len, (blk + 1) * ZERO_BLOCK);
                if (ne > e0 && ext[2 * ne - 2] + ext[2 * ne - 1] == lo) {
                    ext[2 * ne - 1] += hi - lo;
                } else {
                    ext[2 * ne] = lo; ext[2 * ne + 1] = hi - lo;
                    esrc.push_back(u.soff + (lo - u.off));
                    ne++;
                }
                host_bytes += hi - lo;
            }
        }
        ext_first[i + 1] = ne;
    }
    if (ne == 0) return PBSGPU_OK;
    // K14: the data extents, packed per range, through the host-out staging buffer
    Gather ga{b, r, out, nullptr};
    ga.out_dev = false;
    const uint32_t pcap = (uint32_t)std::min<uint64_t>(ne + 1, READER_PIECE_BATCH) * 2;   // a split piece adds one
    ga.d_pieces = b.get<ReadPiece>(pcap);
    ga.d_first = b.get<uint64_t>(pcap + 1);
    ga.pieces.reserve(pcap);
    ga.stage_cap = std::min(host_bytes, READER_STAGE_MAX);
    ga.stage = b.get<uint8_t>(ga.stage_cap);
    if (!ga.d_pieces || !ga.d_first || !ga.stage) return fail(ctx, PBSGPU_ENOMEM, "%s: gather buffers failed", what);
    for (uint32_t i = 0; i < n; i++) {
        uint64_t packed = 0;
        for (uint64_t e = ext_first[i]; e < ext_first[i + 1]; e++) {
            if (int rc = ga.add({0, esrc[e], ext[2 * e + 1], out_off[i] + packed, i, false, false}, dstage)) return rc;
            packed += ext[2 * e + 1];
        }
    }
    return ga.flush();
}

// The sparse image restore's read: the ranges' data chunks (every chunk but the zero chunks) go through
// pbsgpu_reader_read into a device stage owned by this call, K17 maps their 4 KiB block parts that are all zero, and K14
// copies only the data extents of the ranges whose status is OK to the caller's host memory, packed.  Zero chunks
// (zero_chunk) are neither fetched, decoded, cached nor scanned: their block parts are holes by construction.
extern "C" int pbsgpu_reader_read_sparse(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                                         const void *blob_base, const uint64_t *blob_off, const uint64_t *blob_len,
                                         const uint64_t *blob_chunk, uint32_t n_blobs, uint8_t *out, const uint64_t *out_off,
                                         uint64_t *ext, uint64_t ext_cap, uint64_t *ext_first, int32_t *status,
                                         int32_t *blob_status) {
    if (!r || (n && (!off || !len || !out || !out_off || !ext_first || !status)) || (ext_cap && !ext) ||
        (n_blobs && (!blob_base || !blob_off || !blob_len || !blob_chunk)))
        return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = r->ctx;
    Guard g(ctx);
    if (!r->image) return fail(ctx, PBSGPU_EINVAL, "read_sparse: a .didx reader has no sparse read");
    if (int rc = check_ranges(r, off, len, n, flags)) return rc;
    std::vector<uint64_t> bit0;
    if (int rc = sparse_bits(r, off, len, n, out, ext_cap, "read_sparse", bit0)) return rc;
    if (int rc = zero_digests(r)) return rc;
    // the data runs: maximal runs of data chunks within a range; the zero chunks between them are whole blocks
    // (zero_chunk), so every block part lies in one run
    std::vector<SparseRun> runs;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++)
        for_pieces(r, off[i], off[i] + len[i], [&](uint64_t c, uint64_t, uint64_t l, uint64_t at) {
            if (zero_chunk(r, c)) return;
            const uint64_t a = off[i] + at;
            if (!runs.empty() && runs.back().range == i && runs.back().off + runs.back().len == a) {
                runs.back().len += l;
            } else {
                total += (a - total) & 15;
                runs.push_back({a, l, total, i});
            }
            total += l;
        });
    if (runs.size() > UINT32_MAX) return fail(ctx, PBSGPU_EINVAL, "read_sparse: more than 2^32 - 1 data runs");
    const uint32_t nr = (uint32_t)runs.size();
    Blocking b(ctx, ctx->streams[0]);
    uint8_t *dstage = nr ? b.get<uint8_t>(total + 16) : nullptr;
    if (nr && !dstage) return fail(ctx, PBSGPU_ENOMEM, "read_sparse: device stage of %llu bytes failed", (unsigned long long)total);
    std::vector<uint64_t> ro(nr), rl(nr), rs(nr);
    std::vector<int32_t> rst(nr);
    for (uint32_t k = 0; k < nr; k++) { ro[k] = runs[k].off; rl[k] = runs[k].len; rs[k] = runs[k].soff; }
    if (int rc = pbsgpu_reader_read(r, ro.data(), rl.data(), nr, 0, blob_base, blob_off, blob_len, blob_chunk, n_blobs,
                                    dstage, rs.data(), rst.data(), blob_status))
        return rc;
    // a range's status: its first failing data run's (runs are in range order, then chunk order)
    for (uint32_t i = 0; i < n; i++) status[i] = PBSGPU_DEC_OK;
    for (uint32_t k = 0; k < nr; k++)
        if (status[runs[k].range] == PBSGPU_DEC_OK) status[runs[k].range] = rst[k];
    return sparse_extents(r, b, runs, dstage, off, bit0, n, out, out_off, ext, ext_first, status, "read_sparse");
}

// The file restore's read: ranges of pxar file contents, sparse in blocks aligned to each file's content start.  Per
// range, the runs are the data chunks' content bytes widened to whole blocks (clipped to the range) and merged where
// they touch, so runs are apart by at least one whole block that lies in zero chunks.  The stage is zeroed when a run or
// a header spans a zero chunk, then the data chunks' pieces land in it through pbsgpu_reader_read; the 16-byte headers
// of the ranges at pos 0 go to one area after the runs.  The tail is the image form's, with content offsets as block
// coordinates.  Zero chunks (file_zero_chunk) are neither fetched, decoded nor cached.
extern "C" int pbsgpu_reader_read_file_sparse(pbsgpu_reader *r, const uint64_t *file_off, const uint64_t *file_size,
                                              const uint64_t *pos, const uint64_t *len, uint32_t n, const void *blob_base,
                                              const uint64_t *blob_off, const uint64_t *blob_len, const uint64_t *blob_chunk,
                                              uint32_t n_blobs, uint8_t *out, const uint64_t *out_off, uint64_t *ext,
                                              uint64_t ext_cap, uint64_t *ext_first, int32_t *status, int32_t *blob_status) {
    if (!r || (n && (!file_off || !file_size || !pos || !len || !out || !out_off || !ext_first || !status)) ||
        (ext_cap && !ext) || (n_blobs && (!blob_base || !blob_off || !blob_len || !blob_chunk)))
        return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = r->ctx;
    Guard g(ctx);
    if (int rc = check_file_ranges(r, file_off, file_size, pos, len, n)) return rc;
    std::vector<uint64_t> bit0;
    if (int rc = sparse_bits(r, pos, len, n, out, ext_cap, "read_file_sparse", bit0)) return rc;
    if (int rc = zero_digests(r)) return rc;
    // the runs, in content offsets
    std::vector<SparseRun> runs;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t a0 = file_off[i] + 16 + pos[i], end = pos[i] + len[i];
        for_pieces(r, a0, a0 + len[i], [&](uint64_t c, uint64_t, uint64_t l, uint64_t at) {
            if (file_zero_chunk(r, c)) return;
            const uint64_t a = pos[i] + at;
            const uint64_t lo = std::max(pos[i], a / ZERO_BLOCK * ZERO_BLOCK);
            const uint64_t hi = std::min(end, (a + l + ZERO_BLOCK - 1) / ZERO_BLOCK * ZERO_BLOCK);
            if (!runs.empty() && runs.back().range == i && runs.back().off + runs.back().len >= lo)
                runs.back().len = hi - runs.back().off;
            else
                runs.push_back({lo, hi - lo, 0, i});
        });
    }
    if (runs.size() > UINT32_MAX) return fail(ctx, PBSGPU_EINVAL, "read_file_sparse: more than 2^32 - 1 data runs");
    uint64_t total = 0;
    for (SparseRun &u : runs) {
        total += (u.off - total) & 15;
        u.soff = total;
        total += u.len;
    }
    std::vector<uint32_t> hdr_of;   // the ranges at pos 0, in order: their headers at hbase + 16 k
    for (uint32_t i = 0; i < n; i++)
        if (pos[i] == 0) hdr_of.push_back(i);
    const uint64_t hbase = (total + 15) & ~15ull;
    total = hbase + 16 * hdr_of.size();
    // the reads: per range its header, then its runs, each as the maximal runs of data-chunk pieces in it
    struct Read { uint64_t off, len, soff; uint32_t range; };
    std::vector<Read> reads;
    auto stage_span = [&](uint32_t i, uint64_t lo, uint64_t hi, uint64_t soff) {
        for_pieces(r, lo, hi, [&](uint64_t c, uint64_t, uint64_t l, uint64_t at) {
            if (file_zero_chunk(r, c)) return;
            if (!reads.empty() && reads.back().range == i && reads.back().soff + reads.back().len == soff + at &&
                reads.back().off + reads.back().len == lo + at)
                reads.back().len += l;
            else
                reads.push_back({lo + at, l, soff + at, i});
        });
    };
    for (uint32_t i = 0, k = 0, h = 0; i < n; i++) {
        if (pos[i] == 0) stage_span(i, file_off[i], file_off[i] + 16, hbase + 16ull * h++);
        for (; k < runs.size() && runs[k].range == i; k++)
            stage_span(i, file_off[i] + 16 + runs[k].off, file_off[i] + 16 + runs[k].off + runs[k].len, runs[k].soff);
    }
    if (reads.size() > UINT32_MAX) return fail(ctx, PBSGPU_EINVAL, "read_file_sparse: more than 2^32 - 1 data reads");
    const uint32_t nq = (uint32_t)reads.size();
    Blocking b(ctx, ctx->streams[0]);
    uint8_t *dstage = total ? b.get<uint8_t>(total + 16) : nullptr;
    if (total && !dstage) return fail(ctx, PBSGPU_ENOMEM, "read_file_sparse: device stage of %llu bytes failed", (unsigned long long)total);
    uint64_t landed = 0, staged = 16 * hdr_of.size();
    for (const Read &q : reads) landed += q.len;
    for (const SparseRun &u : runs) staged += u.len;
    if (landed < staged) {   // runs or headers span zero chunks: the data pieces land on zeros
        if (b.ok()) b.e = cudaMemsetAsync(dstage, 0, total, b.st);
        if (int rc = b.finish("read_file_sparse stage")) return rc;
    }
    std::vector<uint64_t> ro(nq), rl(nq), rs(nq);
    std::vector<int32_t> rst(nq);
    for (uint32_t k = 0; k < nq; k++) { ro[k] = reads[k].off; rl[k] = reads[k].len; rs[k] = reads[k].soff; }
    if (int rc = pbsgpu_reader_read(r, ro.data(), rl.data(), nq, 0, blob_base, blob_off, blob_len, blob_chunk, n_blobs,
                                    dstage, rs.data(), rst.data(), blob_status))
        return rc;
    // a range's status: its first failing read's (header first, then in archive order), then BAD_HEADER
    for (uint32_t i = 0; i < n; i++) status[i] = PBSGPU_DEC_OK;
    for (uint32_t k = 0; k < nq; k++)
        if (status[reads[k].range] == PBSGPU_DEC_OK) status[reads[k].range] = rst[k];
    if (!hdr_of.empty()) {
        std::vector<uint8_t> hdr(16 * hdr_of.size());
        if (b.ok()) b.e = cudaMemcpyAsync(hdr.data(), dstage + hbase, hdr.size(), cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("read_file_sparse headers")) return rc;
        for (size_t h = 0; h < hdr_of.size(); h++) {
            const uint32_t i = hdr_of[h];
            if (status[i] == PBSGPU_DEC_OK && !payload_header_ok(hdr.data() + 16 * h, file_size[i])) status[i] = PBSGPU_DEC_BAD_HEADER;
        }
    }
    return sparse_extents(r, b, runs, dstage, pos, bit0, n, out, out_off, ext, ext_first, status, "read_file_sparse");
}
