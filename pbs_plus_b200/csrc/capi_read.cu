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
    // sparse calls of an image: the digests of clen zero bytes for the (at most two) chunk lengths, computed on first use
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

// The digests of clen zero bytes for the image's two chunk lengths (chunk_size and the last chunk's), plain or keyed with
// the reader's crypt as the index's digests are: K3 through the SHA-256 batch calls, once per reader.
static int zero_digests(pbsgpu_reader *r) {
    if (r->zero_known || r->ends.empty()) return PBSGPU_OK;
    r->zero_len[0] = r->clen.front();   // the longest: every chunk but the last is chunk_size
    r->zero_len[1] = r->clen.back();
    const std::vector<uint8_t> zeros(r->zero_len[0]);
    const uint64_t at[2] = {0, 0};
    if (int rc = r->crypt ? pbsgpu_sha256_keyed_batch(r->ctx, r->crypt, zeros.data(), at, r->zero_len, 2, r->zero_dig[0])
                          : pbsgpu_sha256_batch(r->ctx, zeros.data(), at, r->zero_len, 2, r->zero_dig[0]))
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
        for (uint32_t i = 0; i < n; i++) {
            uint8_t want[16];
            memcpy(want, PXAR_PAYLOAD_LE, 8);
            for (int k = 0; k < 8; k++) want[8 + k] = (uint8_t)((16 + len[i]) >> (8 * k));
            if (status[i] == PBSGPU_DEC_OK && memcmp(hdr.data() + 16ull * i, want, 16) != 0) status[i] = PBSGPU_DEC_BAD_HEADER;
        }
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
    if (n && pbsgpu_is_device_ptr(out)) return fail(ctx, PBSGPU_EINVAL, "read_sparse: out must be host memory");
    // bit0[i]: the bit of range i's first block part; a range of B block parts has at most ceil(B / 2) extents
    std::vector<uint64_t> bit0(n + 1, 0);
    uint64_t bound = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t parts = len[i] ? (off[i] + len[i] - 1) / ZERO_BLOCK - off[i] / ZERO_BLOCK + 1 : 0;
        bit0[i + 1] = bit0[i] + parts;
        bound += (parts + 1) / 2;
    }
    if (ext_cap < bound)
        return fail(ctx, PBSGPU_EINVAL, "read_sparse: ext_cap %llu < %llu, the most extents the ranges can have",
                    (unsigned long long)ext_cap, (unsigned long long)bound);
    if (int rc = zero_digests(r)) return rc;
    // the data runs: maximal runs of data chunks within a range, staged at offsets congruent to their image offsets
    // mod 16 so K17's vector loads are aligned on whole blocks
    struct Run { uint64_t off, len, soff; uint32_t range; };
    std::vector<Run> runs;
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
    // K17 over the runs of the ranges that are OK
    std::vector<ZeroRun> zr;
    std::vector<uint64_t> part_first(1, 0);
    for (const Run &u : runs) {
        if (status[u.range] != PBSGPU_DEC_OK) continue;
        const uint64_t b0 = u.off / ZERO_BLOCK, b1 = (u.off + u.len - 1) / ZERO_BLOCK;
        zr.push_back({(uint64_t)(uintptr_t)dstage + u.soff, u.off, u.len, bit0[u.range] + b0 - off[u.range] / ZERO_BLOCK});
        part_first.push_back(part_first.back() + b1 - b0 + 1);
    }
    std::vector<uint32_t> bits;
    if (!zr.empty()) {
        const uint64_t words = (bit0[n] + 31) / 32;
        bits.resize(words);
        uint32_t *d_bits = b.get<uint32_t>(words);
        const ZeroRun *d_runs = b.upload(zr.data(), zr.size());
        const uint64_t *d_first = b.upload(part_first.data(), part_first.size());
        if (!d_bits || !d_runs || !d_first) return fail(ctx, PBSGPU_ENOMEM, "read_sparse: zero map buffers failed");
        if (b.ok()) b.e = cudaMemsetAsync(d_bits, 0xff, words * 4, b.st);
        if (b.ok()) b.e = launch_zero_map(d_runs, d_first, (uint32_t)zr.size(), part_first.back(), d_bits, ctx->sm_count, b.st);
        if (b.ok()) b.e = cudaMemcpyAsync(bits.data(), d_bits, words * 4, cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("read_sparse zero map")) return rc;
    }
    // the extents: maximal runs of non-hole block parts.  Two runs of a range are apart by at least one zero chunk whose
    // bounds are block boundaries (zero_chunk), so no block part spans two runs, an extent lies in one run, its dstage
    // bytes are contiguous, and a range has at most ceil(B / 2) extents.
    std::vector<uint64_t> esrc;   // per extent: its offset in dstage
    uint64_t ne = 0, host_bytes = 0;
    if (n) ext_first[0] = 0;
    for (uint32_t i = 0, k = 0; i < n; i++) {
        const uint64_t e0 = ne;
        for (; k < nr && runs[k].range == i; k++) {
            const Run &u = runs[k];
            if (status[i] != PBSGPU_DEC_OK) continue;
            const uint64_t b0 = u.off / ZERO_BLOCK, b1 = (u.off + u.len - 1) / ZERO_BLOCK;
            for (uint64_t blk = b0; blk <= b1; blk++) {
                const uint64_t bit = bit0[i] + blk - off[i] / ZERO_BLOCK;
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
    if (!ga.d_pieces || !ga.d_first || !ga.stage) return fail(ctx, PBSGPU_ENOMEM, "read_sparse gather buffers failed");
    for (uint32_t i = 0; i < n; i++) {
        uint64_t packed = 0;
        for (uint64_t e = ext_first[i]; e < ext_first[i + 1]; e++) {
            if (int rc = ga.add({0, esrc[e], ext[2 * e + 1], out_off[i] + packed, i, false, false}, dstage)) return rc;
            packed += ext[2 * e + 1];
        }
    }
    return ga.flush();
}
