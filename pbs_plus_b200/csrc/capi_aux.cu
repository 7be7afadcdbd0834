// pbs_plus_b200/csrc/capi_aux.cu -- C ABI of the "next" rows of SURVEY.md section 8: dynamic index images (f1), the commit
// walk's per-file XXH3-64 (f2) and DataBlob framing + CRC-32 for new chunks (f3); and the SHA-256 of byte ranges.
// Except for the index images these are blocking calls (host.hpp, Blocking).
#include <errno.h>
#include <sys/random.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "host.hpp"

using namespace pbsgpu;

// ---------------------------------------------------------------------------
// blocking calls: completion, staging of the caller's bytes, constant tables
// ---------------------------------------------------------------------------
int pbsgpu_finish(pbsgpu_ctx *ctx, cudaStream_t st, cudaError_t e, const char *what) {
    const cudaError_t es = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = es;
    if (e == cudaSuccess) return PBSGPU_OK;
    (void)cudaGetLastError();
    return fail(ctx, PBSGPU_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

Blocking::~Blocking() {
    if (blocks.empty()) return;
    if (cudaStreamSynchronize(st) != cudaSuccess) (void)cudaGetLastError();
    for (void *p : blocks) ctx->dev.put(p);
}

int Blocking::stage(const void *base, const uint64_t *off, const uint64_t *len, uint32_t n, const uint8_t **dbase) {
    uint64_t hi = 0;
    for (uint32_t i = 0; i < n; i++) hi = std::max(hi, off[i] + len[i]);
    *dbase = (const uint8_t *)base;
    if (hi == 0 || pbsgpu_is_device_ptr(base)) return PBSGPU_OK;
    uint8_t *p = get<uint8_t>(hi + 16);
    if (!p) return fail(ctx, PBSGPU_ENOMEM, "staging of %llu bytes failed", (unsigned long long)hi);
    *dbase = p;
    if (ok()) e = cudaMemcpyAsync(p, base, hi, cudaMemcpyHostToDevice, st);
    return ok() ? PBSGPU_OK : finish("H2D copy");
}

// K6 / K7 constant tables: built on the host and uploaded on the context's first use (freed with the context)
static int upload_table_once(pbsgpu_ctx *ctx, void **d, size_t bytes, void (*fill)(void *)) {
    if (*d) return PBSGPU_OK;
    std::vector<uint8_t> h(bytes);
    fill(h.data());
    CK(cudaMalloc(d, bytes));
    CK(cudaMemcpy(*d, h.data(), bytes, cudaMemcpyHostToDevice));
    return PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// f1: dynamic index images
// ---------------------------------------------------------------------------
static const uint8_t DIDX_MAGIC[8] = {28, 145, 78, 165, 25, 186, 179, 205};

extern "C" uint64_t pbsgpu_didx_size(uint64_t n) { return 4096 + n * 40; }

extern "C" int pbsgpu_didx_build(pbsgpu_ctx *ctx, const pbsgpu_chunk *chunks, uint64_t n, const uint8_t uuid[16],
                                 int64_t ctime, uint8_t *out, uint64_t cap) {
    if (!ctx || (n && !chunks) || !out || !uuid) return PBSGPU_EINVAL;
    if (cap < pbsgpu_didx_size(n)) return fail(ctx, PBSGPU_ERANGE, "didx buffer too small: %llu < %llu", (unsigned long long)cap, (unsigned long long)pbsgpu_didx_size(n));
    memset(out, 0, 4096);
    memcpy(out, DIDX_MAGIC, 8);
    memcpy(out + 8, uuid, 16);
    for (int i = 0; i < 8; i++) out[24 + i] = (uint8_t)((uint64_t)ctime >> (8 * i));
    uint64_t total = 0, prev_end = 0;
    uint32_t prev_stream = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (i == 0 || chunks[i].stream != prev_stream) prev_end = 0;
        if (chunks[i].end_off < prev_end) return fail(ctx, PBSGPU_EINVAL, "chunk records not ordered by (stream, end_off) at %llu", (unsigned long long)i);
        total += chunks[i].end_off - prev_end;
        prev_end = chunks[i].end_off; prev_stream = chunks[i].stream;
        uint8_t *e = out + 4096 + i * 40;
        for (int k = 0; k < 8; k++) e[k] = (uint8_t)(total >> (8 * k));
        memcpy(e + 8, chunks[i].digest, 32);
    }
    uint64_t off0 = 0, len0 = n * 40;
    return pbsgpu_sha256_batch(ctx, out + 4096, &off0, &len0, 1, out + 32);   // index_csum (GPU)
}

extern "C" int pbsgpu_didx_parse(pbsgpu_ctx *ctx, const uint8_t *didx, uint64_t size, uint64_t *ends, uint8_t *digests,
                                 uint64_t cap, uint64_t *n_entries, int verify) {
    if (!didx || !n_entries) return PBSGPU_EINVAL;
    if (size < 4096 || (size - 4096) % 40 || memcmp(didx, DIDX_MAGIC, 8) != 0)
        return fail(ctx, PBSGPU_EINVAL, "not a dynamic index image");
    uint64_t n = (size - 4096) / 40;
    *n_entries = n;
    if (ends || digests) {
        if (cap < n) return fail(ctx, PBSGPU_ERANGE, "output capacity %llu < %llu entries", (unsigned long long)cap, (unsigned long long)n);
        uint64_t prev = 0;
        for (uint64_t i = 0; i < n; i++) {
            const uint8_t *e = didx + 4096 + i * 40;
            uint64_t end = 0;
            for (int k = 0; k < 8; k++) end |= (uint64_t)e[k] << (8 * k);
            if (end < prev) return fail(ctx, PBSGPU_EINVAL, "index offsets not monotonic at entry %llu", (unsigned long long)i);
            prev = end;
            if (ends) ends[i] = end;
            if (digests) memcpy(digests + i * 32, e + 8, 32);
        }
    }
    if (verify) {
        if (!ctx) return PBSGPU_EINVAL;
        uint8_t csum[32];
        uint64_t off0 = 0, len0 = n * 40;
        int rc = pbsgpu_sha256_batch(ctx, didx + 4096, &off0, &len0, 1, csum);
        if (rc) return rc;
        if (memcmp(csum, didx + 32, 32) != 0) return fail(ctx, PBSGPU_EINVAL, "index checksum mismatch");
    }
    return PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// fixed index images (disk images): header { magic, uuid, ctime, index_csum, size, chunk_size } + the digests
// ---------------------------------------------------------------------------
static const uint8_t FIDX_MAGIC[8] = {0x2f, 0x7f, 0x41, 0xed, 0x91, 0xfd, 0x0f, 0xcd};

static void put_u64(uint8_t *p, uint64_t v) { for (int i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (8 * i)); }
static uint64_t get_u64(const uint8_t *p) { uint64_t v = 0; for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i); return v; }

extern "C" uint64_t pbsgpu_fidx_size(uint64_t n) { return 4096 + n * 32; }

extern "C" int pbsgpu_fidx_build(pbsgpu_ctx *ctx, const uint8_t *digests, uint64_t n, uint64_t size, uint64_t chunk_size,
                                 const uint8_t uuid[16], int64_t ctime, uint8_t *out, uint64_t cap) {
    if (!ctx || (n && !digests) || !out || !uuid) return PBSGPU_EINVAL;
    if (chunk_size == 0 || chunk_size >= (1ull << 32)) return fail(ctx, PBSGPU_EINVAL, "fidx chunk_size %llu not in [1, 2^32)", (unsigned long long)chunk_size);
    if (n != size / chunk_size + (size % chunk_size != 0))
        return fail(ctx, PBSGPU_EINVAL, "fidx: %llu digests for %llu bytes in chunks of %llu", (unsigned long long)n,
                    (unsigned long long)size, (unsigned long long)chunk_size);
    if (cap < pbsgpu_fidx_size(n)) return fail(ctx, PBSGPU_ERANGE, "fidx buffer too small: %llu < %llu", (unsigned long long)cap, (unsigned long long)pbsgpu_fidx_size(n));
    memset(out, 0, 4096);
    memcpy(out, FIDX_MAGIC, 8);
    memcpy(out + 8, uuid, 16);
    put_u64(out + 24, (uint64_t)ctime);
    put_u64(out + 64, size);
    put_u64(out + 72, chunk_size);
    if (n) memcpy(out + 4096, digests, n * 32);
    uint64_t off0 = 0, len0 = n * 32;
    return pbsgpu_sha256_batch(ctx, out + 4096, &off0, &len0, 1, out + 32);   // index_csum (GPU)
}

extern "C" int pbsgpu_fidx_parse(pbsgpu_ctx *ctx, const uint8_t *fidx, uint64_t bytes, uint64_t *size, uint64_t *chunk_size,
                                 uint8_t *digests, uint64_t cap, uint64_t *n_entries, int verify) {
    if (!fidx || !n_entries) return PBSGPU_EINVAL;
    if (bytes < 4096 || memcmp(fidx, FIDX_MAGIC, 8) != 0) return fail(ctx, PBSGPU_EINVAL, "not a fixed index image");
    const uint64_t sz = get_u64(fidx + 64), cs = get_u64(fidx + 72);
    if (cs == 0 || cs >= (1ull << 32)) return fail(ctx, PBSGPU_EINVAL, "fixed index: chunk_size %llu not in [1, 2^32)", (unsigned long long)cs);
    const uint64_t n = sz / cs + (sz % cs != 0);
    if (n > (bytes - 4096) / 32 || bytes - 4096 != n * 32)
        return fail(ctx, PBSGPU_EINVAL, "fixed index: %llu bytes, but size %llu in chunks of %llu needs %llu digests",
                    (unsigned long long)bytes, (unsigned long long)sz, (unsigned long long)cs, (unsigned long long)n);
    *n_entries = n;
    if (size) *size = sz;
    if (chunk_size) *chunk_size = cs;
    if (digests) {
        if (cap < n) return fail(ctx, PBSGPU_ERANGE, "output capacity %llu < %llu entries", (unsigned long long)cap, (unsigned long long)n);
        if (n) memcpy(digests, fidx + 4096, n * 32);
    }
    if (verify) {
        if (!ctx) return PBSGPU_EINVAL;
        uint8_t csum[32];
        uint64_t off0 = 0, len0 = n * 32;
        int rc = pbsgpu_sha256_batch(ctx, fidx + 4096, &off0, &len0, 1, csum);
        if (rc) return rc;
        if (memcmp(csum, fidx + 32, 32) != 0) return fail(ctx, PBSGPU_EINVAL, "index checksum mismatch");
    }
    return PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// SHA-256 of n byte ranges (K3 without the chunker)
// ---------------------------------------------------------------------------
// suffix: encrypt mode's device id_key (keyed digests), or NULL
static int sha256_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                        uint8_t *digests, const uint8_t *suffix) {
    Guard g(ctx);
    if (n == 0) return PBSGPU_OK;
    std::vector<ChunkRef> refs(n);
    for (uint32_t i = 0; i < n; i++) {
        if (len[i] >= (1ull << 32)) return fail(ctx, PBSGPU_EINVAL, "range %u longer than 4 GiB", i);
        refs[i].stream = i; refs[i].len = (uint32_t)len[i]; refs[i].start = off[i];
    }
    Blocking b(ctx, ctx->streams[0]);
    ShaArgs ha;
    if (int rc = b.stage(base, off, len, n, &ha.base)) return rc;
    const unsigned long long hn = n;
    ha.off = nullptr; ha.chunks = b.upload(refs.data(), n); ha.order = nullptr; ha.n_chunks = b.upload(&hn, 1);
    ha.chunk_cap = n; ha.digests = b.get<uint8_t>((uint64_t)n * 32); ha.n_head = nullptr; ha.n_mid = nullptr; ha.part = 0;
    if (!ha.chunks || !ha.n_chunks || !ha.digests) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (b.ok()) b.e = ctx->variant == 1 ? launch_sha_simple(ha, b.st, suffix) : launch_sha_tuned(ha, ctx->tune, b.st, suffix);
    if (b.ok()) b.e = cudaMemcpyAsync(digests, ha.digests, (uint64_t)n * 32, cudaMemcpyDeviceToHost, b.st);
    return b.finish("sha256 batch");
}

extern "C" int pbsgpu_sha256_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len,
                                   uint32_t n, uint8_t *digests) {
    if (!ctx || (n && (!off || !len || !digests))) return PBSGPU_EINVAL;
    return sha256_batch(ctx, base, off, len, n, digests, nullptr);
}

extern "C" int pbsgpu_sha256_keyed_batch(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, const void *base, const uint64_t *off,
                                         const uint64_t *len, uint32_t n, uint8_t *digests) {
    if (!ctx || !crypt || crypt->ctx != ctx || (n && (!off || !len || !digests))) return PBSGPU_EINVAL;
    return sha256_batch(ctx, base, off, len, n, digests, pbsgpu_crypt_id_key(crypt));
}

// ---------------------------------------------------------------------------
// f3: DataBlob checksums
// ---------------------------------------------------------------------------
static const uint8_t BLOB_MAGIC_UNCOMPRESSED[8] = {66, 171, 56, 7, 190, 131, 112, 161};
static const uint8_t BLOB_MAGIC_COMPRESSED[8] = {49, 185, 88, 66, 111, 182, 163, 127};
static const uint8_t BLOB_MAGIC_ENCRYPTED[8] = {0x7b, 0x67, 0x85, 0xbe, 0x22, 0x2d, 0x4c, 0xf0};
static const uint8_t BLOB_MAGIC_ENCR_COMPR[8] = {0xe6, 0x59, 0x1b, 0xbf, 0x0b, 0xbf, 0xd8, 0x0b};

static void blob_header(const uint8_t magic[8], uint32_t crc, uint8_t *out) {
    memcpy(out, magic, 8);
    for (int i = 0; i < 4; i++) out[8 + i] = (uint8_t)(crc >> (8 * i));
}
extern "C" void pbsgpu_blob_header(uint32_t crc, uint8_t out[12]) { blob_header(BLOB_MAGIC_UNCOMPRESSED, crc, out); }

int pbsgpu_crc32_enqueue(Blocking &b, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t *d_out) {
    pbsgpu_ctx *ctx = b.ctx;
    if (int rc = upload_table_once(ctx, &ctx->d_crc_tables, crc_tables_bytes(), crc_fill_tables_host)) return rc;
    const int crc_variant = ctx->crc_variant;   // 0 = TMA-tiled kernel (default), 1 = simple lane-strided kernel (PBSGPU_CRC_VARIANT at open)
    // work units: 128 KiB warp blocks (simple) or <= 576 KiB regions of the 16 B aligned body (tiled)
    const uint64_t UNIT = crc_variant ? crc_wb_bytes() : crc_region_bytes();
    std::vector<uint64_t> wb_first(n + 1);
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        wb_first[i] = total;
        if (crc_variant) total += (len[i] + UNIT - 1) / UNIT;
        else if (len[i]) {
            uint64_t head = (16 - ((uintptr_t)(dbase + off[i]) & 15)) & 15;
            uint64_t body = len[i] > head ? len[i] - head : 0;
            total += std::max<uint64_t>(1, (body + UNIT - 1) / UNIT);
        }
    }
    wb_first[n] = total;
    uint64_t *d_off = b.upload(off, n), *d_len = b.upload(len, n), *d_first = b.upload(wb_first.data(), n + 1);
    uint32_t *d_part = b.get<uint32_t>(total + 1);
    if (!d_off || !d_len || !d_first || !d_part) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (b.ok())
        b.e = crc_variant ? launch_crc32(dbase, d_off, d_len, d_first, n, total, ctx->d_crc_tables, d_part, d_out, ctx->sm_count, b.st)
                          : launch_crc32_tiled(dbase, d_off, d_len, d_first, n, total, ctx->d_crc_tables, d_part, d_out, ctx->sm_count, b.st);
    return PBSGPU_OK;
}

extern "C" int pbsgpu_crc32_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len,
                                  uint32_t n, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !crc_out))) return PBSGPU_EINVAL;
    Guard g(ctx);
    if (n == 0) return PBSGPU_OK;
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    uint32_t *d_out = b.get<uint32_t>(n);
    if (!d_out) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (int rc = pbsgpu_crc32_enqueue(b, dbase, off, len, n, d_out)) return rc;
    if (b.ok()) b.e = cudaMemcpyAsync(crc_out, d_out, (uint64_t)n * 4, cudaMemcpyDeviceToHost, b.st);
    return b.finish("crc32 batch");
}

uint64_t pbsgpu_blob_size_impl(uint64_t payload) { return payload + 12; }
extern "C" uint64_t pbsgpu_blob_size(uint64_t payload_len) { return pbsgpu_blob_size_impl(payload_len); }

// CRC-32 (K6) of the ranges [src + o[i], + l[i]) of the blobs with comp[i] == want, into crc[i]
static int crc_where(pbsgpu_ctx *ctx, const std::vector<uint8_t> &comp, uint8_t want, const void *src, const uint64_t *o,
                     const uint64_t *l, std::vector<uint32_t> &crc) {
    std::vector<uint64_t> so, sl;
    std::vector<uint32_t> idx;
    for (uint32_t i = 0; i < comp.size(); i++) if (comp[i] == want) { idx.push_back(i); so.push_back(o[i]); sl.push_back(l[i]); }
    std::vector<uint32_t> c(idx.size());
    int rc = pbsgpu_crc32_batch(ctx, src, so.data(), sl.data(), (uint32_t)idx.size(), c.data());
    for (size_t k = 0; rc == PBSGPU_OK && k < idx.size(); k++) crc[idx[k]] = c[k];
    return rc;
}

// Which DataBlob encoder a call is: uncompressed only, RLE / raw frames (_z), with the match stage (_lz), with the match
// and entropy stages (_lze), with Huffman literals over every byte value (_lzh), and _lzh with long-distance matches
// across the whole chunk (_lzl).
enum class BlobMode { raw, z, lz, lze, lzh, lzl };
// the encoders by their PBSGPU_BLOB_* value (PBSGPU_BLOB_RAW ..); value 6 is not assigned
static bool blob_mode_of(int mode, BlobMode *m) {
    static const BlobMode modes[] = {BlobMode::raw, BlobMode::z, BlobMode::lz, BlobMode::lze, BlobMode::lzh};
    if (mode >= PBSGPU_BLOB_RAW && mode <= PBSGPU_BLOB_LZH) { *m = modes[mode - PBSGPU_BLOB_RAW]; return true; }
    if (mode == PBSGPU_BLOB_LZL) { *m = BlobMode::lzl; return true; }
    return false;
}

// K12: the long spans of the blocks that are not constant (z = their index in the match stage's list), in order: span
// block y is block span_z[y], with the spans spans[span_first[y] .. span_first[y + 1]) (zlz.cuh's packing).  The kept
// long matches come per pass of whole chunks (LDM_PASS_BYTES, or one longer chunk); each is split at the block edges,
// and pieces in constant blocks or shorter than LZ_MINMATCH are dropped.
static int ldm_spans_of(Blocking &b, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n,
                        const std::vector<uint64_t> &blk_first, const std::vector<int64_t> &zof, std::vector<uint32_t> &span_z,
                        std::vector<uint32_t> &span_first, std::vector<uint64_t> &spans) {
    pbsgpu_ctx *ctx = b.ctx;
    std::vector<uint64_t> sfirst(n + 1), vfirst(n + 1);
    std::vector<uint32_t> pass_c0;
    for (uint32_t i = 0; i < n; i++) {
        sfirst[i + 1] = sfirst[i] + ldm_spans(len[i]);
        vfirst[i + 1] = vfirst[i] + len[i];
    }
    for (uint32_t i = 0; i < n; i++)
        if (pass_c0.empty() || vfirst[i + 1] - vfirst[pass_c0.back()] > LDM_PASS_BYTES || i - pass_c0.back() >= LDM_PASS_CHUNKS)
            pass_c0.push_back(i);
    pass_c0.push_back(n);
    const uint32_t np = (uint32_t)pass_c0.size() - 1;
    if (sfirst[n] == 0) return PBSGPU_OK;
    uint64_t *d_sfirst = b.upload(sfirst.data(), n + 1), *d_vfirst = b.upload(vfirst.data(), n + 1);
    uint64_t *d_off = b.upload(off, n), *d_len = b.upload(len, n);
    unsigned long long *d_tot = b.get<unsigned long long>(np);
    if (!d_sfirst || !d_vfirst || !d_off || !d_len || !d_tot) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    auto pass = [&](uint32_t p) {
        const uint32_t c0 = pass_c0[p], c1 = pass_c0[p + 1];
        return LdmArgs{dbase, d_off, d_len, d_sfirst, d_vfirst, c0, c1, sfirst[c0], sfirst[c1]};
    };
    // K12a over every pass: the anchor counts size the scratch
    std::vector<unsigned long long> tot(np);
    if (b.ok()) b.e = cudaMemsetAsync(d_tot, 0, np * sizeof(unsigned long long), b.st);
    for (uint32_t p = 0; b.ok() && p < np; p++) b.e = launch_ldm_count(pass(p), d_tot + p, b.st);
    if (b.ok()) b.e = cudaMemcpyAsync(tot.data(), d_tot, np * sizeof(unsigned long long), cudaMemcpyDeviceToHost, b.st);
    if (int rc = b.finish("ldm anchor count")) return rc;
    size_t scratch_bytes = 0;
    for (uint32_t p = 0; p < np; p++) {
        if (tot[p] >= (1ull << 31)) return fail(ctx, PBSGPU_EINVAL, "more than 2^31 long-match anchors in one chunk");
        scratch_bytes = std::max(scratch_bytes, ldm_scratch_bytes(pass(p).s1 - pass(p).s0, tot[p]));
    }
    uint8_t *scratch = b.get<uint8_t>(scratch_bytes);
    if (!scratch) return fail(ctx, PBSGPU_ENOMEM, "long-match scratch of %llu bytes failed", (unsigned long long)scratch_bytes);
    // K12 per pass; the kept matches as (chunk, start, end, offset)
    struct Kept { uint64_t chunk, s, e, d; };
    std::vector<Kept> kept;
    std::vector<uint64_t> hk, hv;
    for (uint32_t p = 0; p < np; p++) {
        if (tot[p] < 2) continue;
        uint64_t *dk, *dv;
        uint32_t *dn, nk = 0;
        b.e = launch_ldm_matches(pass(p), tot[p], scratch, &dk, &dv, &dn, b.st);
        if (b.ok()) b.e = cudaMemcpyAsync(&nk, dn, 4, cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("ldm matches")) return rc;
        hk.resize(nk); hv.resize(nk);
        if (nk && b.ok()) b.e = cudaMemcpyAsync(hk.data(), dk, nk * 8ull, cudaMemcpyDeviceToHost, b.st);
        if (nk && b.ok()) b.e = cudaMemcpyAsync(hv.data(), dv, nk * 8ull, cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("ldm matches")) return rc;
        for (uint32_t k = 0; k < nk; k++)
            kept.push_back({pass_c0[p] + (hk[k] >> 40), hk[k] & LDM_M40, hv[k] & LDM_M40, hv[k] >> 40});
    }
    std::sort(kept.begin(), kept.end(), [](const Kept &x, const Kept &y) { return x.chunk != y.chunk ? x.chunk < y.chunk : x.s < y.s; });
    span_first.assign(1, 0);
    for (const Kept &m : kept) {
        for (uint64_t k = m.s / ZFRAME_BLOCK; k <= (m.e - 1) / ZFRAME_BLOCK; k++) {
            const uint64_t ps = std::max<uint64_t>(m.s, k * ZFRAME_BLOCK), pe = std::min<uint64_t>(m.e, (k + 1) * ZFRAME_BLOCK);
            const int64_t z = zof[blk_first[m.chunk] + k];
            if (z < 0 || pe - ps < LZ_MINMATCH) continue;
            if (span_z.empty() || span_z.back() != (uint32_t)z) { span_z.push_back((uint32_t)z); span_first.push_back(span_first.back()); }
            spans.push_back((ps - k * ZFRAME_BLOCK) | (pe - ps) << 20 | m.d << 40);
            span_first.back()++;
        }
    }
    return PBSGPU_OK;
}

// Compressed form: a blob's payload is a zstd frame when that is smaller than the raw bytes (upstream
// `DataBlob::encode` keeps the compressed form only then).  The frame is built on the device (zframe.cu, zlz.cu,
// zent.cu): a 128 KiB block of one repeated byte is an RLE_Block (K8a decides); with lz / lze / lzh every other block
// goes through the match stage (K9; lze and lzh add the entropy stage, K10, lzh with its full-alphabet flag) and is a
// Compressed_Block when that is smaller than the block; the rest are Raw_Blocks.  The CRC (K6) covers the frame.  Marks those blobs in comp[] and leaves their frames at *frames + frame_off[i] (frame_len[i] bytes, a block
// of `b`) and their CRCs in crc[].
static int zstd_frames(Blocking &b, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n, BlobMode mode,
                       std::vector<uint8_t> &comp, std::vector<uint64_t> &frame_off, std::vector<uint64_t> &frame_len,
                       std::vector<uint32_t> &crc, const uint8_t **frames) {
    pbsgpu_ctx *ctx = b.ctx;
    // K8a: which 128 KiB blocks are one repeated byte
    std::vector<uint64_t> blk_first(n + 1);
    uint64_t n_blocks = 0;
    for (uint32_t i = 0; i < n; i++) { blk_first[i] = n_blocks; n_blocks += (len[i] + ZFRAME_BLOCK - 1) / ZFRAME_BLOCK; }
    blk_first[n] = n_blocks;
    if (n_blocks >= (1ull << 31)) return fail(ctx, PBSGPU_EINVAL, "too many 128 KiB blocks in one call (%llu)", (unsigned long long)n_blocks);
    std::vector<uint32_t> flags(n_blocks);
    uint64_t *d_off = b.upload(off, n), *d_len = b.upload(len, n), *d_first = b.upload(blk_first.data(), n + 1);
    uint32_t *d_flags = b.get<uint32_t>(n_blocks + 1);
    if (!d_off || !d_len || !d_first || !d_flags) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (b.ok()) b.e = launch_zblock_scan(dbase, d_off, d_len, d_first, n, n_blocks, d_flags, b.st);
    if (b.ok() && n_blocks) b.e = cudaMemcpyAsync(flags.data(), d_flags, n_blocks * 4, cudaMemcpyDeviceToHost, b.st);
    if (int rc = b.finish("zstd block scan")) return rc;
    auto block_size = [&](uint32_t i, uint64_t k) { return (uint32_t)std::min<uint64_t>(ZFRAME_BLOCK, len[i] - k * ZFRAME_BLOCK); };
    // K9 (+ K10): the match stage and encoding of the blocks that are not constant, in passes of LZ_PASS_BLOCKS.  With
    // lzl, K12 first finds the long spans; the blocks that hold one are parsed again with them (K9a's span parse, K9b,
    // K10) into slots nz + y, and each such block keeps the smaller content, K9's on ties.
    const bool ent = mode == BlobMode::lze || mode == BlobMode::lzh || mode == BlobMode::lzl, lz = mode == BlobMode::lz || ent;
    const bool full = mode == BlobMode::lzh || mode == BlobMode::lzl;
    std::vector<uint32_t> info;
    std::vector<uint64_t> slot_of;   // the slot of block z's content
    const uint8_t *slots = nullptr;
    if (lz) {
        std::vector<uint64_t> zsrc;
        std::vector<uint32_t> zsize;
        std::vector<int64_t> zof(n_blocks, -1);
        for (uint32_t i = 0; i < n; i++)
            for (uint64_t k = 0; k < blk_first[i + 1] - blk_first[i]; k++)
                if (!(flags[blk_first[i] + k] & 0x100u)) {
                    zof[blk_first[i] + k] = (int64_t)zsrc.size();
                    zsrc.push_back(off[i] + k * ZFRAME_BLOCK); zsize.push_back(block_size(i, k));
                }
        const uint64_t nz = zsrc.size();
        std::vector<uint32_t> span_z, span_first;
        std::vector<uint64_t> spans;
        if (mode == BlobMode::lzl && nz)
            if (int rc = ldm_spans_of(b, dbase, off, len, n, blk_first, zof, span_z, span_first, spans)) return rc;
        const uint64_t ny = span_z.size();
        for (uint64_t y = 0; y < ny; y++) { zsrc.push_back(zsrc[span_z[y]]); zsize.push_back(zsize[span_z[y]]); }
        if (nz) {
            if (int rc = upload_table_once(ctx, &ctx->d_lz_tab, sizeof(LzTables), lz_fill_tables_host)) return rc;
            const uint64_t nall = nz + ny;
            uint64_t *d_zsrc = b.upload(zsrc.data(), nall);
            uint32_t *d_zsize = b.upload(zsize.data(), nall);
            uint8_t *d_slots = b.get<uint8_t>(nall * LZ_SLOT);
            uint64_t *d_seqs = b.get<uint64_t>(std::min<uint64_t>(nall, LZ_PASS_BLOCKS) * LZ_MAX_SEQ);
            uint32_t *d_nseq = b.get<uint32_t>(nall), *d_nlit = b.get<uint32_t>(nall), *d_info = b.get<uint32_t>(nall);
            uint8_t *d_ent = ent ? b.get<uint8_t>(std::min<uint64_t>(nall, LZ_PASS_BLOCKS) * ENT_SCRATCH) : nullptr;
            uint64_t *d_spans = ny ? b.upload(spans.data(), spans.size()) : nullptr;
            uint32_t *d_span_first = ny ? b.upload(span_first.data(), ny + 1) : nullptr;
            if (!d_zsrc || !d_zsize || !d_slots || !d_seqs || !d_nseq || !d_nlit || !d_info || (ent && !d_ent) ||
                (ny && (!d_spans || !d_span_first)))
                return fail(ctx, PBSGPU_ENOMEM, "match stage: device allocation failed");
            // the blocks [0, nz), then the span blocks [nz, nz + ny), each list in passes of its own
            auto passes = [&](uint64_t lo, uint64_t hi, bool span_parse) {
                for (uint64_t f = lo; b.ok() && f < hi; f += LZ_PASS_BLOCKS) {
                    const uint32_t pn = (uint32_t)std::min<uint64_t>(LZ_PASS_BLOCKS, hi - f);
                    b.e = span_parse ? launch_lz_parse_spans(dbase, d_zsrc, d_zsize, f, pn, d_slots, d_seqs, d_nseq, d_nlit,
                                                             d_spans, d_span_first, nz, b.st)
                                     : launch_lz_parse(dbase, d_zsrc, d_zsize, f, pn, d_slots, d_seqs, d_nseq, d_nlit, b.st);
                    if (b.ok()) b.e = launch_lz_encode((const LzTables *)ctx->d_lz_tab, f, pn, d_slots, d_seqs, d_nseq, d_nlit, d_info, b.st);
                    if (b.ok() && d_ent)
                        b.e = launch_ent_encode((const LzTables *)ctx->d_lz_tab, d_zsize, f, pn, d_slots, d_seqs, d_nseq, d_nlit,
                                                d_info, d_ent, full, b.st);
                }
            };
            passes(0, nz, false);
            passes(nz, nall, true);
            info.resize(nall);
            if (b.ok()) b.e = cudaMemcpyAsync(info.data(), d_info, nall * 4, cudaMemcpyDeviceToHost, b.st);
            if (int rc = b.finish("zstd match stage")) return rc;
            slots = d_slots;
            slot_of.resize(nz);
            for (uint64_t z = 0; z < nz; z++) slot_of[z] = z;
            for (uint64_t y = 0; y < ny; y++)   // a span block keeps its span parse when that is smaller
                if ((info[nz + y] & 0x3FFFFFFFu) < (info[span_z[y]] & 0x3FFFFFFFu)) slot_of[span_z[y]] = nz + y;
        }
    }
    // every block's Block_Header (bits 0..23; the RLE byte in 24..31), body size and body source (dbase + src, or
    // slots + src for a Compressed_Block)
    std::vector<uint32_t> bhdr(n_blocks), bbody(n_blocks);
    std::vector<uint64_t> bsrc(n_blocks);
    for (uint32_t i = 0, z = 0; i < n; i++) {
        const uint64_t nb = blk_first[i + 1] - blk_first[i];
        for (uint64_t k = 0; k < nb; k++) {
            const uint64_t blk = blk_first[i] + k;
            const uint32_t size = block_size(i, k), f = flags[blk], last = k + 1 == nb;
            uint32_t type = 0, hsize = size, body = size;
            bsrc[blk] = off[i] + k * ZFRAME_BLOCK;
            if (f & 0x100u) { type = 1; body = 1; }
            else if (lz) {
                const uint64_t y = slot_of[z];
                const uint32_t cs = info[y] & 0x3FFFFFFFu;
                if (cs < size) { type = 2; hsize = body = cs; bsrc[blk] = y * LZ_SLOT + (info[y] >> 30); }
                z++;
            }
            bhdr[blk] = last | type << 1 | hsize << 3 | (f & 0xFFu) << 24;
            bbody[blk] = body;
        }
    }
    // frame sizes; the blobs that come out smaller get a place in the stage and one emit entry per block, in the list of
    // their body's source
    std::vector<uint64_t> foff, content, e_src[2], e_dst[2];
    std::vector<uint32_t> e_hdr[2];
    uint64_t cursor = 0;
    for (uint32_t i = 0; i < n; i++) {
        uint64_t fl = ZFRAME_HEADER;
        for (uint64_t blk = blk_first[i]; blk < blk_first[i + 1]; blk++) fl += 3 + bbody[blk];
        if (len[i] == 0 || fl >= len[i]) continue;
        comp[i] = 1; frame_off[i] = cursor; frame_len[i] = fl;
        foff.push_back(cursor);
        content.push_back(len[i]);
        uint64_t pos = cursor + ZFRAME_HEADER;
        for (uint64_t blk = blk_first[i]; blk < blk_first[i + 1]; blk++) {
            const int from_slot = ((bhdr[blk] >> 1) & 3) == 2;
            e_src[from_slot].push_back(bsrc[blk]);
            e_dst[from_slot].push_back(pos);
            e_hdr[from_slot].push_back(bhdr[blk]);
            pos += 3 + bbody[blk];
        }
        cursor = (pos + 15) & ~15ull;
    }
    const uint32_t nc = (uint32_t)foff.size();
    if (nc == 0) return PBSGPU_OK;
    uint8_t *stage = b.get<uint8_t>(cursor + 16);
    if (!stage) return fail(ctx, PBSGPU_ENOMEM, "frame staging of %llu bytes failed", (unsigned long long)cursor);
    uint64_t *d_foff = b.upload(foff.data(), nc), *d_clen = b.upload(content.data(), nc);
    if (!d_foff || !d_clen) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (b.ok()) b.e = launch_zframe_hdr(stage, d_foff, d_clen, nc, b.st);
    for (int s = 0; s < 2; s++) {
        const uint64_t ne = e_hdr[s].size();
        if (ne == 0) continue;
        uint64_t *d_src = b.upload(e_src[s].data(), ne), *d_dst = b.upload(e_dst[s].data(), ne);
        uint32_t *d_hdr = b.upload(e_hdr[s].data(), ne);
        if (!d_src || !d_dst || !d_hdr) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
        if (b.ok()) b.e = launch_zframe_emit(s ? slots : dbase, stage, d_src, d_dst, d_hdr, ne, b.st);
    }
    if (int rc = b.finish("zstd frame emit")) return rc;
    *frames = stage;
    return crc_where(ctx, comp, 1, stage, frame_off.data(), frame_len.data(), crc);
}

// f3: complete DataBlobs for the NEW chunks of a batch in one call (upstream pbs-datastore data_blob.rs:
// magic[8] | crc32 LE over the payload | payload; uploaded by POST /dynamic_chunk, reference
// internal/server/backup/log_cleanup.go:19-31), with zstd frames as payloads where they are smaller unless `mode` is
// raw.
// The CRCs come from K6 on the device; payload bytes are copied once (device -> host for resident data and frames,
// host -> host otherwise) straight into their place behind the header.
static int blob_encode(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n, BlobMode mode,
                       uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    Guard g(ctx);
    const bool compress = mode != BlobMode::raw;
    if (n == 0) return PBSGPU_OK;
    for (uint32_t i = 0; compress && i < n; i++)
        if (len[i] >= (1ull << 40)) return fail(ctx, PBSGPU_EINVAL, "blob %u longer than 2^40 bytes", i);
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase, *frames = nullptr;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    std::vector<uint8_t> comp(n, 0);
    std::vector<uint64_t> frame_off(n), frame_len(n);
    std::vector<uint32_t> crc(n, 0);
    if (compress) {
        int rc = zstd_frames(b, dbase, off, len, n, mode, comp, frame_off, frame_len, crc, &frames);
        if (rc) return rc;
    }
    if (int rc = crc_where(ctx, comp, 0, dbase, off, len, crc)) return rc;
    // assemble in the caller's memory; staged payloads are copied from the caller's host memory
    const bool staged = dbase != (const uint8_t *)base;
    cudaError_t e = cudaSuccess;
    for (uint32_t i = 0; i < n && e == cudaSuccess; i++) {
        uint8_t *blob = out + out_off[i];
        blob_header(comp[i] ? BLOB_MAGIC_COMPRESSED : BLOB_MAGIC_UNCOMPRESSED, crc[i], blob);
        const uint64_t plen = comp[i] ? frame_len[i] : len[i];
        if (out_len) out_len[i] = 12 + plen;
        if (plen == 0) continue;
        if (comp[i]) e = cudaMemcpyAsync(blob + 12, frames + frame_off[i], plen, cudaMemcpyDeviceToHost, ctx->copy_stream);
        else if (staged) memcpy(blob + 12, (const uint8_t *)base + off[i], plen);
        else e = cudaMemcpyAsync(blob + 12, dbase + off[i], plen, cudaMemcpyDeviceToHost, ctx->copy_stream);
    }
    if (int rc = pbsgpu_finish(ctx, ctx->copy_stream, e, "blob assembly copy")) return rc;
    if (crc_out) memcpy(crc_out, crc.data(), (size_t)n * 4);
    return PBSGPU_OK;
}

// The stream's blob mode (capi_stream.cu): one of the PBSGPU_BLOB_* encoders.
int pbsgpu_blob_encode_mode(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n, int mode,
                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len) {
    BlobMode m;
    if (!blob_mode_of(mode, &m)) return fail(ctx, PBSGPU_EINVAL, "unknown blob mode %d", mode);
    return blob_encode(ctx, base, off, len, n, m, out, out_off, out_len, nullptr);
}

extern "C" int pbsgpu_blob_encode_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                        uint8_t *out, const uint64_t *out_off, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !base))) return PBSGPU_EINVAL;
    return blob_encode(ctx, base, off, len, n, BlobMode::raw, out, out_off, nullptr, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_z(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                          uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !out_len || !base))) return PBSGPU_EINVAL;
    return blob_encode(ctx, base, off, len, n, BlobMode::z, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lz(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                           uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !out_len || !base))) return PBSGPU_EINVAL;
    return blob_encode(ctx, base, off, len, n, BlobMode::lz, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lze(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !out_len || !base))) return PBSGPU_EINVAL;
    return blob_encode(ctx, base, off, len, n, BlobMode::lze, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lzh(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !out_len || !base))) return PBSGPU_EINVAL;
    return blob_encode(ctx, base, off, len, n, BlobMode::lzh, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lzl(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || !out_len || !base))) return PBSGPU_EINVAL;
    return blob_encode(ctx, base, off, len, n, BlobMode::lzl, out, out_off, out_len, crc_out);
}

// ---------------------------------------------------------------------------
// f3, read side: decode and verify DataBlobs (K6, K11, K13, K3)
// ---------------------------------------------------------------------------
// The blobs are staged once; K6 takes the CRC of every payload.  Then, per pass of whole blobs (at most ZDEC_PASS_BLOBS
// blobs, ZDEC_PASS_BYTES decoded bytes and ZDEC_PASS_BYTES of ciphertext, or one longer blob), K13 decodes into the
// caller's device buffer or a pass buffer, K3 hashes the chunks that decoded, and a host `out` receives those chunks
// from the pass buffer.  The host reads only statuses and digests back; no decoded byte crosses PCIe unless `out` is
// host memory.
// With crypt, the host first reads every blob's header and sorts the blobs by magic.  Bad magics and encrypted blobs
// whose CRC (K6 over the ciphertext) differs stop there.  Per pass, K11 decrypts the other encrypted payloads into a
// plaintext stage, laid out as plain blobs (zdec.cuh), and the host compares their tags; K13 then decodes the plain
// blobs from the input and the authenticated ones from the stage, so no unauthenticated byte reaches `out`.  K3 hashes
// the chunks of encrypted blobs keyed with the crypt's id_key, the others plain (upstream `DataBlob::decode` with a
// config).  Without crypt nothing is read on the host and every blob goes to K13 from the input.
int pbsgpu_blob_decode(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, const void *base, const uint64_t *off, const uint64_t *len,
                       uint32_t n, const uint64_t *chunk_len, const uint8_t *digest, uint8_t *out, const uint64_t *out_off,
                       int32_t *status, uint8_t *digest_out) {
    Guard g(ctx);
    if (n == 0) return PBSGPU_OK;
    for (uint32_t i = 0; i < n; i++) {
        if (chunk_len[i] >= (1ull << 32)) return fail(ctx, PBSGPU_EINVAL, "chunk %u: chunk_len >= 2^32", i);
        if (off[i] + len[i] < off[i]) return fail(ctx, PBSGPU_EINVAL, "blob %u: range wraps around", i);
    }
    if (int rc = upload_table_once(ctx, &ctx->d_zdec_tab, sizeof(ZdecTables), zdec_fill_tables_host)) return rc;
    const bool out_dev = out && pbsgpu_is_device_ptr(out), want_sha = digest || digest_out;
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    // kind[i]: the magic's index in BLOB_MAGICS (K13's order), -1 for an unknown magic or a blob shorter than its header;
    // without crypt every blob is left to K13 (0).  heads: the first ZDEC_HEAD bytes of every blob.
    static const uint8_t *const BLOB_MAGICS[4] = {BLOB_MAGIC_UNCOMPRESSED, BLOB_MAGIC_COMPRESSED, BLOB_MAGIC_ENCRYPTED,
                                                  BLOB_MAGIC_ENCR_COMPR};
    std::vector<int8_t> kind(n, 0);
    std::vector<uint8_t> heads;
    if (crypt) {
        heads.assign((size_t)n * ZDEC_HEAD, 0);
        if (!pbsgpu_is_device_ptr(base)) {   // host base: read in place
            for (uint32_t i = 0; i < n; i++)
                memcpy(heads.data() + (size_t)ZDEC_HEAD * i, (const uint8_t *)base + off[i], std::min<uint64_t>(len[i], ZDEC_HEAD));
        } else {
            uint64_t *d_off = b.upload(off, n), *d_len = b.upload(len, n);
            uint8_t *d_heads = b.get<uint8_t>((uint64_t)n * ZDEC_HEAD);
            if (!d_off || !d_len || !d_heads) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
            if (b.ok()) b.e = launch_blob_heads(dbase, d_off, d_len, n, d_heads, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(heads.data(), d_heads, heads.size(), cudaMemcpyDeviceToHost, b.st);
            if (int rc = b.finish("blob headers")) return rc;
        }
        for (uint32_t i = 0; i < n; i++) {
            kind[i] = -1;
            for (int m = 0; m < 4 && kind[i] < 0; m++)
                if (memcmp(heads.data() + (size_t)ZDEC_HEAD * i, BLOB_MAGICS[m], 8) == 0) kind[i] = (int8_t)m;
            if (kind[i] >= 0 && len[i] < (kind[i] >= 2 ? ZDEC_HEAD : 12)) kind[i] = -1;
        }
    }
    // K6 over the payloads: [12, len) of a plain blob, [44, len) of an encrypted one (a blob too short for its header
    // gets an empty range; its magic check fails first).  ct[i]: the ciphertext bytes of an encrypted blob.
    std::vector<uint64_t> poff(n), plen(n), ct(n, 0);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t hs = kind[i] >= 2 ? ZDEC_HEAD : 12;
        poff[i] = off[i] + hs; plen[i] = len[i] >= hs ? len[i] - hs : 0;
        if (kind[i] >= 2) ct[i] = plen[i];
    }
    uint32_t *d_crc = b.get<uint32_t>(n);
    if (!d_crc) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (int rc = pbsgpu_crc32_enqueue(b, dbase, poff.data(), plen.data(), n, d_crc)) return rc;
    std::vector<uint32_t> crc;
    if (crypt) {   // the host checks the magics and the CRCs of encrypted blobs; K13 those of plain blobs
        crc.resize(n);
        if (b.ok()) b.e = cudaMemcpyAsync(crc.data(), d_crc, n * 4ull, cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("blob crc")) return rc;
        for (uint32_t i = 0; i < n; i++) {
            const uint8_t *h = heads.data() + (size_t)ZDEC_HEAD * i;
            const uint32_t hc = (uint32_t)h[8] | (uint32_t)h[9] << 8 | (uint32_t)h[10] << 16 | (uint32_t)h[11] << 24;
            status[i] = kind[i] < 0 ? PBSGPU_DEC_BAD_MAGIC : kind[i] >= 2 && hc != crc[i] ? PBSGPU_DEC_BAD_CRC : PBSGPU_DEC_OK;
        }
    }
    // passes of whole blobs
    std::vector<uint32_t> pass_first;
    uint64_t pass_max = 0, acc = 0, acc_c = 0, blobs_max = 0, stage_max = 0, stage_acc = 0, segs_max = 0, segs_acc = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (pass_first.empty() || acc + chunk_len[i] > ZDEC_PASS_BYTES || acc_c + ct[i] > ZDEC_PASS_BYTES ||
            i - pass_first.back() >= ZDEC_PASS_BLOBS) {
            pass_first.push_back(i);
            acc = acc_c = stage_acc = segs_acc = 0;
        }
        acc += chunk_len[i];
        acc_c += ct[i];
        if (kind[i] >= 2) { stage_acc += 16 + ((ct[i] + 15) & ~15ull); segs_acc += gcm_segments(ct[i]); }
        pass_max = std::max(pass_max, acc);
        stage_max = std::max(stage_max, stage_acc);
        segs_max = std::max(segs_max, segs_acc);
        blobs_max = std::max<uint64_t>(blobs_max, i - pass_first.back() + 1);
    }
    pass_first.push_back(n);
    uint8_t *pbuf = out_dev ? nullptr : b.get<uint8_t>(pass_max + 16);
    uint8_t *lits = b.get<uint8_t>(blobs_max * ZDEC_LIT_SLOT);
    ZdecBlob *d_blobs = b.get<ZdecBlob>(blobs_max);
    int32_t *d_status = b.get<int32_t>(blobs_max);
    ChunkRef *d_refs = want_sha ? b.get<ChunkRef>(blobs_max) : nullptr;
    unsigned long long *d_nref = want_sha ? b.get<unsigned long long>(1) : nullptr;
    uint8_t *d_dig = want_sha ? b.get<uint8_t>(blobs_max * 32) : nullptr;
    if ((!out_dev && !pbuf) || !lits || !d_blobs || !d_status || (want_sha && (!d_refs || !d_nref || !d_dig)))
        return fail(ctx, PBSGPU_ENOMEM, "decode pass buffers (%llu bytes) failed", (unsigned long long)pass_max);
    // encrypt mode: the plaintext stage and K11's buffers, per pass
    uint8_t *stage = nullptr, *d_part = nullptr, *d_tags = nullptr, *d_shead = nullptr;
    GcmMsg *d_msg = nullptr;
    uint64_t *d_first = nullptr, *d_sat = nullptr;
    uint32_t *d_csub = nullptr;
    if (crypt) {
        stage = b.get<uint8_t>(stage_max + 16); d_part = b.get<uint8_t>(segs_max * 16 + 16);
        d_tags = b.get<uint8_t>(blobs_max * 16); d_shead = b.get<uint8_t>(blobs_max * 16);
        d_msg = b.get<GcmMsg>(blobs_max); d_first = b.get<uint64_t>(blobs_max + 1); d_sat = b.get<uint64_t>(blobs_max);
        d_csub = b.get<uint32_t>(blobs_max);
        if (!stage || !d_part || !d_tags || !d_shead || !d_msg || !d_first || !d_sat || !d_csub)
            return fail(ctx, PBSGPU_ENOMEM, "decryption stage (%llu bytes) failed", (unsigned long long)stage_max);
    }
    std::vector<ZdecBlob> zb(blobs_max);
    std::vector<uint64_t> at(blobs_max), sat(blobs_max);   // chunk k of the pass at pass base + at[k]; its plaintext blob at stage + sat[k]
    std::vector<ChunkRef> refs(blobs_max);
    std::vector<uint32_t> ref_blob(blobs_max), list(blobs_max), csub(blobs_max);
    std::vector<int32_t> st(blobs_max);
    std::vector<uint8_t> dig(blobs_max * 32), tags, shead;
    std::vector<GcmMsg> msg;
    std::vector<uint64_t> seg_first;
    for (size_t p = 0; p + 1 < pass_first.size(); p++) {
        const uint32_t i0 = pass_first[p], pn = pass_first[p + 1] - i0;
        uint8_t *pbase = out_dev ? out : pbuf;
        uint64_t cur = 0, scur = 0;
        for (uint32_t k = 0; k < pn; k++) {   // the caller's places, or back to back in the pass buffer
            const uint32_t i = i0 + k;
            at[k] = out_dev ? out_off[i] : cur;
            cur += chunk_len[i];
            sat[k] = scur;
            if (kind[i] >= 2) scur += 16 + ((ct[i] + 15) & ~15ull);
        }
        // K11: the encrypted payloads whose CRC matched, decrypted into the stage; their tags compared on the host in
        // constant time (XOR-accumulate)
        msg.clear(); seg_first.assign(1, 0); list.clear();
        for (uint32_t k = 0; crypt && k < pn; k++) {
            const uint32_t i = i0 + k;
            if (kind[i] < 2 || status[i] != PBSGPU_DEC_OK) continue;
            GcmMsg m;
            m.src = (uint64_t)(uintptr_t)(dbase + off[i] + ZDEC_HEAD);
            m.dst = (uint64_t)(uintptr_t)(stage + sat[k] + 16);
            m.len = ct[i];
            gcm_j0_host(crypt->tab.data(), heads.data() + (size_t)ZDEC_HEAD * i + 12, m.j0);
            gcm_encrypt_block_host(crypt->tab.data(), m.j0, m.ej0);
            msg.push_back(m);
            seg_first.push_back(seg_first.back() + gcm_segments(ct[i]));
            list.push_back(k);
        }
        if (!msg.empty()) {
            const uint32_t ne = (uint32_t)msg.size();
            tags.resize(16ull * ne);
            if (b.ok()) b.e = cudaMemcpyAsync(d_msg, msg.data(), ne * sizeof(GcmMsg), cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(d_first, seg_first.data(), (ne + 1) * 8ull, cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = launch_gcm(d_msg, d_first, ne, seg_first[ne], crypt->d_tab, d_part, d_tags, ctx->sm_count, b.st, true);
            if (b.ok()) b.e = cudaMemcpyAsync(tags.data(), d_tags, 16ull * ne, cudaMemcpyDeviceToHost, b.st);
            if (int rc = b.finish("blob decryption")) return rc;
            for (uint32_t r = 0; r < ne; r++) {
                const uint32_t i = i0 + list[r];
                const uint8_t *want = heads.data() + (size_t)ZDEC_HEAD * i + 28;
                uint8_t diff = 0;
                for (int j = 0; j < 16; j++) diff |= (uint8_t)(tags[16ull * r + j] ^ want[j]);
                if (diff) status[i] = PBSGPU_DEC_BAD_TAG;
            }
        }
        // K13, once over the plain blobs against the input and once over the authenticated ones against the stage, each
        // behind a plain header (the magic of the payload's form, the CRC K13 is given)
        list.clear(); shead.clear();
        uint32_t n_plain = 0;
        for (int from_stage = 0; from_stage < 2; from_stage++)
            for (uint32_t k = 0; k < pn; k++) {
                const uint32_t i = i0 + k;
                if (crypt && (status[i] != PBSGPU_DEC_OK || (kind[i] >= 2) != (from_stage == 1))) continue;
                if (!crypt && from_stage) break;
                const uint32_t r = (uint32_t)list.size();
                list.push_back(k);
                const uint64_t dst = (uint64_t)(uintptr_t)(pbase + at[k]);
                if (from_stage) {
                    zb[r] = {sat[k] + 4, 12 + ct[i], dst, chunk_len[i]};
                    uint8_t h[16] = {0};
                    blob_header(BLOB_MAGICS[kind[i] - 2], crc[i], h + 4);
                    shead.insert(shead.end(), h, h + 16);
                } else {
                    zb[r] = {off[i], len[i], dst, chunk_len[i]};
                    n_plain++;
                }
                if (crypt) csub[r] = crc[i];
            }
        const uint32_t nl = (uint32_t)list.size(), n_stage = nl - n_plain;
        const uint32_t *crc_l = crypt ? d_csub : d_crc + i0;
        if (b.ok() && nl) b.e = cudaMemcpyAsync(d_blobs, zb.data(), nl * sizeof(ZdecBlob), cudaMemcpyHostToDevice, b.st);
        if (b.ok() && crypt && nl) b.e = cudaMemcpyAsync(d_csub, csub.data(), nl * 4ull, cudaMemcpyHostToDevice, b.st);
        if (n_stage) {
            std::vector<uint64_t> sat_l(n_stage);
            for (uint32_t r = 0; r < n_stage; r++) sat_l[r] = sat[list[n_plain + r]];
            if (b.ok()) b.e = cudaMemcpyAsync(d_sat, sat_l.data(), n_stage * 8ull, cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(d_shead, shead.data(), shead.size(), cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = launch_stage_heads(stage, d_sat, d_shead, n_stage, b.st);
        }
        const ZdecTables *ztab = (const ZdecTables *)ctx->d_zdec_tab;
        if (b.ok()) b.e = launch_zdec(dbase, d_blobs, crc_l, n_plain, ztab, lits, d_status, b.st);
        if (b.ok()) b.e = launch_zdec(stage, d_blobs + n_plain, crc_l + n_plain, n_stage, ztab, lits, d_status + n_plain, b.st);
        if (b.ok() && nl) b.e = cudaMemcpyAsync(st.data(), d_status, nl * sizeof(int32_t), cudaMemcpyDeviceToHost, b.st);
        if (int rc = b.finish("blob decode")) return rc;
        for (uint32_t r = 0; r < nl; r++) status[i0 + list[r]] = st[r];
        // K3 over the chunks that decoded: plain digests, then keyed ones for the encrypted blobs
        for (int keyed = 0; want_sha && keyed < 2; keyed++) {
            uint32_t nr = 0;
            for (uint32_t k = 0; k < pn; k++)
                if (status[i0 + k] == PBSGPU_DEC_OK && (kind[i0 + k] >= 2) == (keyed == 1)) {
                    refs[nr].stream = nr; refs[nr].len = (uint32_t)chunk_len[i0 + k]; refs[nr].start = at[k];
                    ref_blob[nr++] = i0 + k;
                }
            if (nr == 0) continue;
            const uint8_t *suffix = keyed ? pbsgpu_crypt_id_key(crypt) : nullptr;
            const unsigned long long hn = nr;
            ShaArgs ha;
            ha.base = pbase; ha.off = nullptr; ha.chunks = d_refs; ha.order = nullptr; ha.n_chunks = d_nref;
            ha.chunk_cap = nr; ha.digests = d_dig; ha.n_head = nullptr; ha.n_mid = nullptr; ha.part = 0;
            if (b.ok()) b.e = cudaMemcpyAsync(d_refs, refs.data(), nr * sizeof(ChunkRef), cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(d_nref, &hn, sizeof hn, cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = ctx->variant == 1 ? launch_sha_simple(ha, b.st, suffix) : launch_sha_tuned(ha, ctx->tune, b.st, suffix);
            if (b.ok()) b.e = cudaMemcpyAsync(dig.data(), d_dig, nr * 32ull, cudaMemcpyDeviceToHost, b.st);
            if (int rc = b.finish("blob decode digests")) return rc;
            for (uint32_t r = 0; r < nr; r++) {
                const uint32_t i = ref_blob[r];
                if (digest_out) memcpy(digest_out + 32ull * i, dig.data() + 32ull * r, 32);
                if (digest && memcmp(digest + 32ull * i, dig.data() + 32ull * r, 32) != 0) status[i] = PBSGPU_DEC_BAD_DIGEST;
            }
        }
        // a host `out` receives the chunks that decoded
        if (out && !out_dev) {
            for (uint32_t k = 0; b.ok() && k < pn; k++) {
                const uint32_t i = i0 + k;
                if ((status[i] == PBSGPU_DEC_OK || status[i] == PBSGPU_DEC_BAD_DIGEST) && chunk_len[i])
                    b.e = cudaMemcpyAsync(out + out_off[i], pbuf + at[k], chunk_len[i], cudaMemcpyDeviceToHost, b.st);
            }
            if (int rc = b.finish("blob decode copy")) return rc;
        }
    }
    return PBSGPU_OK;
}

extern "C" int pbsgpu_blob_decode_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                        const uint64_t *chunk_len, const uint8_t *digest, uint8_t *out, const uint64_t *out_off,
                                        int32_t *status, uint8_t *digest_out) {
    if (!ctx || (n && (!base || !off || !len || !chunk_len || !status || (out && !out_off)))) return PBSGPU_EINVAL;
    return pbsgpu_blob_decode(ctx, nullptr, base, off, len, n, chunk_len, digest, out, out_off, status, digest_out);
}

extern "C" int pbsgpu_blob_decode_batch_enc(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, const void *base, const uint64_t *off,
                                            const uint64_t *len, uint32_t n, const uint64_t *chunk_len, const uint8_t *digest,
                                            uint8_t *out, const uint64_t *out_off, int32_t *status, uint8_t *digest_out) {
    if (!ctx || !crypt || crypt->ctx != ctx || (n && (!base || !off || !len || !chunk_len || !status || (out && !out_off))))
        return PBSGPU_EINVAL;
    return pbsgpu_blob_decode(ctx, crypt, base, off, len, n, chunk_len, digest, out, out_off, status, digest_out);
}

// ---------------------------------------------------------------------------
// f3, encrypt mode: encrypted DataBlobs (K11)
// ---------------------------------------------------------------------------

// Host SHA-256 (FIPS 180-4) for the key derivation: 20 compressions per crypt handle, so no device work
struct HostSha256 {
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    uint8_t buf[64];
    uint64_t n = 0;
    static uint32_t ror(uint32_t x, int r) { return (x >> r) | (x << (32 - r)); }
    void block(const uint8_t *p) {
        static const uint32_t K[64] = {
            0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
            0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
            0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
            0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
            0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
            0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
            0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
        uint32_t w[64], v[8];
        for (int i = 0; i < 16; i++) w[i] = (uint32_t)p[4 * i] << 24 | (uint32_t)p[4 * i + 1] << 16 | (uint32_t)p[4 * i + 2] << 8 | p[4 * i + 3];
        for (int i = 16; i < 64; i++)
            w[i] = w[i - 16] + (ror(w[i - 15], 7) ^ ror(w[i - 15], 18) ^ (w[i - 15] >> 3)) + w[i - 7] +
                   (ror(w[i - 2], 17) ^ ror(w[i - 2], 19) ^ (w[i - 2] >> 10));
        memcpy(v, h, sizeof v);
        for (int i = 0; i < 64; i++) {
            const uint32_t t1 = v[7] + (ror(v[4], 6) ^ ror(v[4], 11) ^ ror(v[4], 25)) + ((v[4] & v[5]) ^ (~v[4] & v[6])) + K[i] + w[i];
            const uint32_t t2 = (ror(v[0], 2) ^ ror(v[0], 13) ^ ror(v[0], 22)) + ((v[0] & v[1]) ^ (v[0] & v[2]) ^ (v[1] & v[2]));
            memmove(v + 1, v, 7 * sizeof(uint32_t));
            v[4] += t1; v[0] = t1 + t2;
        }
        for (int i = 0; i < 8; i++) h[i] += v[i];
    }
    void update(const uint8_t *p, size_t len) {
        for (size_t i = 0; i < len; i++) { buf[n++ & 63] = p[i]; if ((n & 63) == 0) block(buf); }
    }
    void final(uint8_t out[32]) {
        const uint64_t bits = n * 8;
        const uint8_t one = 0x80, zero = 0;
        update(&one, 1);
        while ((n & 63) != 56) update(&zero, 1);
        for (int i = 7; i >= 0; i--) { const uint8_t b = (uint8_t)(bits >> (8 * i)); update(&b, 1); }
        for (int i = 0; i < 8; i++) for (int k = 0; k < 4; k++) out[4 * i + k] = (uint8_t)(h[i] >> (24 - 8 * k));
    }
};
static void hmac_sha256(const uint8_t key[32], const uint8_t *msg, size_t len, uint8_t out[32]) {
    uint8_t pad[64], inner[32];
    HostSha256 a, b;
    for (int i = 0; i < 64; i++) pad[i] = (uint8_t)((i < 32 ? key[i] : 0) ^ 0x36);
    a.update(pad, 64); a.update(msg, len); a.final(inner);
    for (int i = 0; i < 64; i++) pad[i] ^= 0x36 ^ 0x5c;
    b.update(pad, 64); b.update(inner, 32); b.final(out);
}
// upstream CryptConfig::new: id_key = PBKDF2-HMAC-SHA256(key, "_id_key", 10 iterations, 32 bytes) -- one output block
static void derive_id_key(const uint8_t key[32], uint8_t out[32]) {
    const uint8_t salt[11] = {'_', 'i', 'd', '_', 'k', 'e', 'y', 0, 0, 0, 1};   // salt || INT(1)
    uint8_t u[32], t[32];
    hmac_sha256(key, salt, sizeof salt, u);
    memcpy(t, u, 32);
    for (int it = 1; it < 10; it++) {
        hmac_sha256(key, u, 32, u);
        for (int i = 0; i < 32; i++) t[i] ^= u[i];
    }
    memcpy(out, t, 32);
    volatile uint8_t *z = u;
    for (int i = 0; i < 32; i++) z[i] = 0, t[i] = 0;
}

int pbsgpu_stream_ivs(pbsgpu_ctx *ctx, const uint8_t *seed, uint64_t first, uint32_t n, uint8_t *iv) {
    if (!seed) {
        for (size_t got = 0; got < 16ull * n;) {
            const ssize_t r = getrandom(iv + got, 16ull * n - got, 0);
            if (r < 0 && errno != EINTR) return fail(ctx, PBSGPU_EINVAL, "getrandom failed: %s", strerror(errno));
            if (r > 0) got += (size_t)r;
        }
        return PBSGPU_OK;
    }
    for (uint32_t i = 0; i < n; i++) {
        uint8_t msg[40], d[32];
        memcpy(msg, seed, 32);
        for (int k = 0; k < 8; k++) msg[32 + k] = (uint8_t)((first + i) >> (8 * k));
        HostSha256 h;
        h.update(msg, sizeof msg);
        h.final(d);
        memcpy(iv + 16ull * i, d, 16);
    }
    return PBSGPU_OK;
}

extern "C" int pbsgpu_crypt_create(pbsgpu_ctx *ctx, const uint8_t key[32], pbsgpu_crypt **out) {
    if (!ctx || !key || !out) return PBSGPU_EINVAL;
    Guard g(ctx);
    pbsgpu_crypt *c = new pbsgpu_crypt{ctx, std::vector<uint8_t>(gcm_tables_bytes() + 32), nullptr};
    gcm_fill_tables_host(key, c->tab.data());
    derive_id_key(key, c->tab.data() + gcm_tables_bytes());
    cudaError_t e = cudaMalloc((void **)&c->d_tab, c->tab.size());
    if (e == cudaSuccess) e = cudaMemcpy(c->d_tab, c->tab.data(), c->tab.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        pbsgpu_crypt_destroy(c);
        return fail(ctx, PBSGPU_ECUDA, "crypt tables: %s", cudaGetErrorString(e));
    }
    *out = c;
    return PBSGPU_OK;
}

extern "C" void pbsgpu_crypt_destroy(pbsgpu_crypt *c) {
    if (!c) return;
    Guard g(c->ctx);
    if (c->d_tab) {
        if (cudaMemset(c->d_tab, 0, c->tab.size()) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) (void)cudaGetLastError();
        cudaFree(c->d_tab);
    }
    volatile uint8_t *p = c->tab.data();   // volatile: the zeroing of memory that is freed next is not optimised away
    for (size_t i = 0; i < c->tab.size(); i++) p[i] = 0;
    delete c;
}

extern "C" uint64_t pbsgpu_blob_size_enc(uint64_t payload_len) { return payload_len + 44; }

// The payloads as blob_encode chooses them (zstd_frames for the compressing modes), encrypted by K11 from where they lie
// (the caller's device memory, the H2D stage or the frame stage) into a new stage; K6 over the ciphertext; the blobs are
// assembled in the caller's memory as blob_encode does.
extern "C" int pbsgpu_blob_encode_batch_enc(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, int mode, const void *base,
                                            const uint64_t *off, const uint64_t *len, uint32_t n, const uint8_t *iv,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    BlobMode bm;
    if (!ctx || !crypt || crypt->ctx != ctx || !blob_mode_of(mode, &bm) ||
        (n && (!off || !len || !iv || !out || !out_off || !out_len || !base)))
        return PBSGPU_EINVAL;
    Guard g(ctx);
    if (n == 0) return PBSGPU_OK;
    for (uint32_t i = 0; i < n; i++)
        if (len[i] >= (1ull << 36)) return fail(ctx, PBSGPU_EINVAL, "blob %u longer than 2^36 bytes", i);
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase, *frames = nullptr;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    std::vector<uint8_t> comp(n, 0);
    std::vector<uint64_t> frame_off(n), frame_len(n);
    std::vector<uint32_t> crc(n, 0);
    if (bm != BlobMode::raw)
        if (int rc = zstd_frames(b, dbase, off, len, n, bm, comp, frame_off, frame_len, crc, &frames)) return rc;
    // K11: payload i -> stage + c_off[i] (16 B aligned), tag i
    std::vector<GcmMsg> msg(n);
    std::vector<uint64_t> seg_first(n + 1), c_off(n), c_len(n);
    uint64_t cursor = 0, segs = 0;
    for (uint32_t i = 0; i < n; i++) {
        c_len[i] = comp[i] ? frame_len[i] : len[i];
        c_off[i] = cursor;
        cursor += (c_len[i] + 15) & ~15ull;
        seg_first[i] = segs;
        segs += gcm_segments(c_len[i]);
        msg[i].src = (uint64_t)(uintptr_t)(comp[i] ? frames + frame_off[i] : dbase + off[i]);
        msg[i].len = c_len[i];
        gcm_j0_host(crypt->tab.data(), iv + 16ull * i, msg[i].j0);
        gcm_encrypt_block_host(crypt->tab.data(), msg[i].j0, msg[i].ej0);
    }
    seg_first[n] = segs;
    uint8_t *stage = b.get<uint8_t>(cursor + 16);
    if (!stage) return fail(ctx, PBSGPU_ENOMEM, "ciphertext staging of %llu bytes failed", (unsigned long long)cursor);
    for (uint32_t i = 0; i < n; i++) msg[i].dst = (uint64_t)(uintptr_t)(stage + c_off[i]);
    GcmMsg *d_msg = b.upload(msg.data(), n);
    uint64_t *d_first = b.upload(seg_first.data(), n + 1);
    uint8_t *d_part = b.get<uint8_t>(segs * 16 + 16), *d_tags = b.get<uint8_t>(16ull * n);
    if (!d_msg || !d_first || !d_part || !d_tags) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    std::vector<uint8_t> tags(16ull * n);
    if (b.ok()) b.e = launch_gcm(d_msg, d_first, n, segs, crypt->d_tab, d_part, d_tags, ctx->sm_count, b.st);
    if (b.ok()) b.e = cudaMemcpyAsync(tags.data(), d_tags, 16ull * n, cudaMemcpyDeviceToHost, b.st);
    if (int rc = b.finish("aes-256-gcm")) return rc;
    if (int rc = pbsgpu_crc32_batch(ctx, stage, c_off.data(), c_len.data(), n, crc.data())) return rc;
    cudaError_t e = cudaSuccess;
    for (uint32_t i = 0; i < n && e == cudaSuccess; i++) {
        uint8_t *blob = out + out_off[i];
        blob_header(comp[i] ? BLOB_MAGIC_ENCR_COMPR : BLOB_MAGIC_ENCRYPTED, crc[i], blob);
        memcpy(blob + 12, iv + 16ull * i, 16);
        memcpy(blob + 28, tags.data() + 16ull * i, 16);
        out_len[i] = 44 + c_len[i];
        if (c_len[i]) e = cudaMemcpyAsync(blob + 44, stage + c_off[i], c_len[i], cudaMemcpyDeviceToHost, ctx->copy_stream);
    }
    if (int rc = pbsgpu_finish(ctx, ctx->copy_stream, e, "blob assembly copy")) return rc;
    if (crc_out) memcpy(crc_out, crc.data(), (size_t)n * 4);
    return PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// f2: XXH3-64 of n byte ranges (the commit walk's per-file content hash, commit.go:717-725, :957-976).
// Blocks are hashed in passes of at most PBSGPU_XXH3_CAP_BLOCKS (default 8 Mi = 8 GiB of input, 512 MiB
// of per-block sums); a pass takes the same block window of EVERY stream so the chains stay parallel.
// xxh3_enqueue only enqueues (all passes, no host wait) so the fused batch call can put it on a job's
// stream; xxh3_collect waits for the stream and brings the n hashes back.
// ---------------------------------------------------------------------------

void pbsgpu_xxh3_release(pbsgpu_ctx *ctx, XxhRun *r) {
    ctx->dev.put(r->d_off); ctx->dev.put(r->d_len); ctx->dev.put(r->d_first); ctx->dev.put(r->d_out);
    ctx->dev.put(r->d_state); ctx->dev.put(r->d_S);
    *r = XxhRun();
}

int pbsgpu_xxh3_table(pbsgpu_ctx *ctx, const void **tab) {
    const int rc = upload_table_once(ctx, &ctx->d_xxh_tab, xxh3_tables_bytes(), xxh3_fill_tables_host);
    *tab = ctx->d_xxh_tab;
    return rc;
}

int pbsgpu_xxh3_enqueue(pbsgpu_ctx *ctx, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n,
                        cudaStream_t st, XxhRun *r) {
    if (int rc = upload_table_once(ctx, &ctx->d_xxh_tab, xxh3_tables_bytes(), xxh3_fill_tables_host)) return rc;
    const uint64_t cap_blocks = ctx->xxh3_cap_blocks;
    uint64_t total_all = 0, max_nb = 0, n_long = 0;
    std::vector<uint64_t> nb(n);
    for (uint32_t i = 0; i < n; i++) {
        nb[i] = len[i] > 240 ? (len[i] - 1) >> 10 : 0;
        total_all += nb[i]; max_nb = std::max(max_nb, nb[i]); n_long += nb[i] != 0;
    }
    const bool one = total_all <= cap_blocks;
    const uint64_t win = one ? std::max<uint64_t>(max_nb, 1) : std::max<uint64_t>(1, cap_blocks / n_long);
    const uint64_t s_blocks = one ? total_all : std::min(total_all, n_long * win);
    const uint64_t passes = (max_nb + win - 1) / win;
    r->n = n;
    r->d_off = (uint64_t *)ctx->dev.get(n * 8); r->d_len = (uint64_t *)ctx->dev.get(n * 8);
    r->d_first = (uint64_t *)ctx->dev.get(std::max<uint64_t>(passes, 1) * (n + 1) * 8);
    r->d_out = (uint64_t *)ctx->dev.get((uint64_t)n * 8); r->d_state = (uint64_t *)ctx->dev.get((uint64_t)n * 64);
    r->d_S = (uint64_t *)ctx->dev.get(std::max<uint64_t>(s_blocks, 1) * 64);
    if (!r->d_off || !r->d_len || !r->d_first || !r->d_out || !r->d_state || !r->d_S) {
        pbsgpu_xxh3_release(ctx, r);
        return fail(ctx, PBSGPU_ENOMEM, "xxh3: device allocation failed");
    }
    cudaError_t e = cudaMemcpyAsync(r->d_off, off, n * 8, cudaMemcpyHostToDevice, st);   // pageable sources are staged before return
    if (e == cudaSuccess) e = cudaMemcpyAsync(r->d_len, len, n * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = launch_xxh3_small(dbase, r->d_off, r->d_len, n, ctx->d_xxh_tab, r->d_out, st);
    std::vector<uint64_t> first(n + 1);
    uint64_t pass = 0;
    for (uint64_t lo = 0; e == cudaSuccess && lo < max_nb; lo += win, pass++) {
        uint64_t total = 0;
        for (uint32_t i = 0; i < n; i++) {
            first[i] = total;
            if (nb[i] > lo) total += std::min(nb[i] - lo, win);
        }
        first[n] = total;
        uint64_t *df = r->d_first + pass * (n + 1);
        e = cudaMemcpyAsync(df, first.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = launch_xxh3_pass(dbase, r->d_off, r->d_len, df, n, total, lo, win, ctx->d_xxh_tab, r->d_S, r->d_state, r->d_out, st);
    }
    if (e == cudaSuccess) return PBSGPU_OK;
    const int rc = pbsgpu_finish(ctx, st, e, "xxh3");   // the run's blocks go back once the stream is idle
    pbsgpu_xxh3_release(ctx, r);
    return rc;
}

int pbsgpu_xxh3_collect(pbsgpu_ctx *ctx, XxhRun *r, uint64_t *hash_out, cudaStream_t st) {
    if (!r->d_out) return PBSGPU_OK;
    const int rc = pbsgpu_finish(ctx, st, cudaMemcpyAsync(hash_out, r->d_out, (uint64_t)r->n * 8, cudaMemcpyDeviceToHost, st), "xxh3");
    pbsgpu_xxh3_release(ctx, r);
    return rc;
}

extern "C" int pbsgpu_xxh3_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len,
                                 uint32_t n, uint64_t *hash_out) {
    if (!ctx || (n && (!off || !len || !hash_out))) return PBSGPU_EINVAL;
    Guard g(ctx);
    if (n == 0) return PBSGPU_OK;
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    XxhRun run;
    const int rc = pbsgpu_xxh3_enqueue(ctx, dbase, off, len, n, b.st, &run);
    return rc ? rc : pbsgpu_xxh3_collect(ctx, &run, hash_out, b.st);
}
