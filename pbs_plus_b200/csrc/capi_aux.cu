// pbs_plus_b200/csrc/capi_aux.cu -- C ABI of the "next" rows of SURVEY.md section 8: dynamic and fixed index images
// (f1), the commit walk's per-file XXH3-64 (f2) and the SHA-256 and CRC-32 of byte ranges; and the plumbing of every
// blocking call (host.hpp, Blocking).  Except for the index images these are blocking calls.
#include <algorithm>
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

int pbsgpu_upload_table_once(pbsgpu_ctx *ctx, void **d, size_t bytes, void (*fill)(void *)) {
    if (*d) return PBSGPU_OK;
    std::vector<uint8_t> h(bytes);
    fill(h.data());
    CK(cudaMalloc(d, bytes));
    CK(cudaMemcpy(*d, h.data(), bytes, cudaMemcpyHostToDevice));
    return PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// index images: a 4096-byte header { magic, uuid, ctime, index_csum, ... } and the entries behind it (the body)
// ---------------------------------------------------------------------------
static const uint8_t DIDX_MAGIC[8] = {28, 145, 78, 165, 25, 186, 179, 205};
static const uint8_t FIDX_MAGIC[8] = {0x2f, 0x7f, 0x41, 0xed, 0x91, 0xfd, 0x0f, 0xcd};

static void put_u64(uint8_t *p, uint64_t v) { for (int i = 0; i < 8; i++) p[i] = (uint8_t)(v >> (8 * i)); }
static uint64_t get_u64(const uint8_t *p) { uint64_t v = 0; for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i); return v; }

static void index_header(uint8_t *out, const uint8_t magic[8], const uint8_t uuid[16], int64_t ctime) {
    memset(out, 0, 4096);
    memcpy(out, magic, 8);
    memcpy(out + 8, uuid, 16);
    put_u64(out + 24, (uint64_t)ctime);
}

// index_csum: the SHA-256 (GPU) of the image's body of `body` bytes.  Build writes it to `out` (the header's bytes
// 32..64); parse passes NULL and checks it against those bytes.
static int index_csum(pbsgpu_ctx *ctx, const uint8_t *img, uint64_t body, uint8_t *out) {
    if (!ctx) return PBSGPU_EINVAL;
    uint8_t csum[32];
    uint64_t off0 = 0;
    if (int rc = pbsgpu_sha256_batch(ctx, img + 4096, &off0, &body, 1, out ? out : csum)) return rc;
    return out || memcmp(csum, img + 32, 32) == 0 ? PBSGPU_OK : fail(ctx, PBSGPU_EINVAL, "index checksum mismatch");
}

// f1: dynamic index images, entries { end offset, digest }
extern "C" uint64_t pbsgpu_didx_size(uint64_t n) { return 4096 + n * 40; }

extern "C" int pbsgpu_didx_build(pbsgpu_ctx *ctx, const pbsgpu_chunk *chunks, uint64_t n, const uint8_t uuid[16],
                                 int64_t ctime, uint8_t *out, uint64_t cap) {
    if (!ctx || (n && !chunks) || !out || !uuid) return PBSGPU_EINVAL;
    if (cap < pbsgpu_didx_size(n)) return fail(ctx, PBSGPU_ERANGE, "didx buffer too small: %llu < %llu", (unsigned long long)cap, (unsigned long long)pbsgpu_didx_size(n));
    index_header(out, DIDX_MAGIC, uuid, ctime);
    uint64_t total = 0, prev_end = 0;
    uint32_t prev_stream = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (i == 0 || chunks[i].stream != prev_stream) prev_end = 0;
        if (chunks[i].end_off < prev_end) return fail(ctx, PBSGPU_EINVAL, "chunk records not ordered by (stream, end_off) at %llu", (unsigned long long)i);
        total += chunks[i].end_off - prev_end;
        prev_end = chunks[i].end_off; prev_stream = chunks[i].stream;
        uint8_t *e = out + 4096 + i * 40;
        put_u64(e, total);
        memcpy(e + 8, chunks[i].digest, 32);
    }
    return index_csum(ctx, out, n * 40, out + 32);
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
            const uint64_t end = get_u64(e);
            if (end < prev) return fail(ctx, PBSGPU_EINVAL, "index offsets not monotonic at entry %llu", (unsigned long long)i);
            prev = end;
            if (ends) ends[i] = end;
            if (digests) memcpy(digests + i * 32, e + 8, 32);
        }
    }
    return verify ? index_csum(ctx, didx, n * 40, nullptr) : PBSGPU_OK;
}

// fixed index images (disk images): the header adds { size, chunk_size } at 64; entries are digests
extern "C" uint64_t pbsgpu_fidx_size(uint64_t n) { return 4096 + n * 32; }

extern "C" int pbsgpu_fidx_build(pbsgpu_ctx *ctx, const uint8_t *digests, uint64_t n, uint64_t size, uint64_t chunk_size,
                                 const uint8_t uuid[16], int64_t ctime, uint8_t *out, uint64_t cap) {
    if (!ctx || (n && !digests) || !out || !uuid) return PBSGPU_EINVAL;
    if (chunk_size == 0 || chunk_size >= (1ull << 32)) return fail(ctx, PBSGPU_EINVAL, "fidx chunk_size %llu not in [1, 2^32)", (unsigned long long)chunk_size);
    if (n != size / chunk_size + (size % chunk_size != 0))
        return fail(ctx, PBSGPU_EINVAL, "fidx: %llu digests for %llu bytes in chunks of %llu", (unsigned long long)n,
                    (unsigned long long)size, (unsigned long long)chunk_size);
    if (cap < pbsgpu_fidx_size(n)) return fail(ctx, PBSGPU_ERANGE, "fidx buffer too small: %llu < %llu", (unsigned long long)cap, (unsigned long long)pbsgpu_fidx_size(n));
    index_header(out, FIDX_MAGIC, uuid, ctime);
    put_u64(out + 64, size);
    put_u64(out + 72, chunk_size);
    if (n) memcpy(out + 4096, digests, n * 32);
    return index_csum(ctx, out, n * 32, out + 32);
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
    return verify ? index_csum(ctx, fidx, n * 32, nullptr) : PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// SHA-256 of n byte ranges (K3 without the chunker)
// ---------------------------------------------------------------------------
void pbsgpu_sha256_enqueue(Blocking &b, const uint8_t *base, const ChunkRef *d_refs, const unsigned long long *d_n, uint32_t n,
                           const uint8_t *suffix, uint8_t *d_dig) {
    const ShaArgs ha{base, nullptr, d_refs, nullptr, d_n, n, d_dig, nullptr, 0};
    if (b.ok()) b.e = b.ctx->variant == 1 ? launch_sha_simple(ha, b.st, suffix) : launch_sha_tuned(ha, b.st, suffix);
}

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
    const uint8_t *dbase;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    const unsigned long long hn = n;
    const ChunkRef *d_refs = b.upload(refs.data(), n);
    const unsigned long long *d_n = b.upload(&hn, 1);
    uint8_t *d_dig = b.get<uint8_t>((uint64_t)n * 32);
    if (!d_refs || !d_n || !d_dig) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    pbsgpu_sha256_enqueue(b, dbase, d_refs, d_n, n, suffix, d_dig);
    if (b.ok()) b.e = cudaMemcpyAsync(digests, d_dig, (uint64_t)n * 32, cudaMemcpyDeviceToHost, b.st);
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
// f3: CRC-32 of n byte ranges (K6; DataBlob checksums)
// ---------------------------------------------------------------------------
int pbsgpu_crc32_enqueue(Blocking &b, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t *d_out) {
    pbsgpu_ctx *ctx = b.ctx;
    if (int rc = pbsgpu_upload_table_once(ctx, &ctx->d_crc_tables, crc_tables_bytes(), crc_fill_tables_host)) return rc;
    // work units: <= 576 KiB regions of the 16 B aligned body, at least one per non-empty range
    const uint64_t UNIT = crc_region_bytes();
    std::vector<uint64_t> region_first(n + 1);
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        region_first[i] = total;
        if (len[i]) {
            uint64_t head = (16 - ((uintptr_t)(dbase + off[i]) & 15)) & 15;
            uint64_t body = len[i] > head ? len[i] - head : 0;
            total += std::max<uint64_t>(1, (body + UNIT - 1) / UNIT);
        }
    }
    region_first[n] = total;
    uint64_t *d_off = b.upload(off, n), *d_len = b.upload(len, n), *d_first = b.upload(region_first.data(), n + 1);
    uint32_t *d_part = b.get<uint32_t>(total + 1);
    if (!d_off || !d_len || !d_first || !d_part) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    if (b.ok()) b.e = launch_crc32_tiled(dbase, d_off, d_len, d_first, n, total, ctx->d_crc_tables, d_part, d_out, ctx->sm_count, b.st);
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
    const int rc = pbsgpu_upload_table_once(ctx, &ctx->d_xxh_tab, xxh3_tables_bytes(), xxh3_fill_tables_host);
    *tab = ctx->d_xxh_tab;
    return rc;
}

int pbsgpu_xxh3_enqueue(pbsgpu_ctx *ctx, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n,
                        cudaStream_t st, XxhRun *r) {
    if (int rc = pbsgpu_upload_table_once(ctx, &ctx->d_xxh_tab, xxh3_tables_bytes(), xxh3_fill_tables_host)) return rc;
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
