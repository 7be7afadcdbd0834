// pbs_plus_b200/csrc/capi_stream.cu -- streaming form of the C ABI (pbsgpu_stream_*).
//
// Mirrors how the reference feeds ONE io.Reader of known size through the chunker: transfer.ArchiveWriter.
// WriteEntryReader(entry, io.Reader, size) at internal/pxarmount/commit.go:718-720 (scan() state carried across reads),
// and -- with pbsgpu_stream_suggest -- the archive PAYLOAD stream the production chunker actually sees (16-byte PAYLOAD
// header + content per file, concatenated; pxarfs.go:408-411).
//
// Data path: bytes enter through a pinned staging ring owned by the stream (reserve -> the caller reads straight into
// it -> commit) or through write(), and travel to the current device window with asynchronous copies on the context's
// copy stream: nothing waits per write.  When a window (default 2 GiB) is full its scan + resolve run at once (the host
// needs the cut points to know which tail is still undecided and must be carried into the next window), the carry is
// copied device-to-device behind the scan, and the window's SHA-256 half is enqueued asynchronously -- so the serial tail
// of a window's longest chunk overlaps the copies and scans of the following windows (up to PBSGPU_STREAM_NBUF in
// flight).  poll() hands out the chunks of finished windows in stream order.
//
// Two optional products of a window, made before its buffer is released:
//  - DataBlobs of its new chunks (pbsgpu_stream_blob_mode): at collect time the window's chunks without
//    PBSGPU_CHUNK_KNOWN are encoded in place by the batch encoder (capi_blob.cu) into a pinned arena of the stream.
//  - XXH3-64 of registered byte ranges (pbsgpu_stream_hash_range): each window hashes the blocks, tails and short ranges
//    that lie in its CONSUMED part [base_off, base_off + consumed) with K7's piece form, on the stream's own CUDA stream
//    (window k+1 continues window k's chain).  Ranges do not overlap, so at most one range crosses a window end; the
//    span of it that is still needed (a block, the tail or a short range: < 1 KiB) is copied device-to-device into the
//    carry area in front of the next window's buffer, which makes it contiguous with the window's bytes.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <deque>

#include "host.hpp"

using namespace pbsgpu;

// The hash work of one window: the pinned lists it was launched with (its results come back behind them), the device
// block of lists, block sums and results, and the registration indices of the ranges it finishes.
struct WindowHash {
    void *host = nullptr, *dev = nullptr;
    const uint64_t *h_out = nullptr;   // [n] hashes of the window's ranges
    std::vector<uint64_t> seq;         // registration index of every range finished here ...
    std::vector<uint32_t> slot;        // ... and its index in the window's list
    cudaEvent_t done = nullptr;
};
struct StreamJob { pbsgpu_job *j; int buf; uint64_t base_off; WindowHash *wh; };
struct BlobWindow { uint8_t *host; std::vector<uint64_t> off, len; size_t next; };   // one window's blobs, back to back
struct HashRange { uint64_t off, len, h; bool done; };
constexpr int RING_SLOTS = 8;
constexpr uint64_t CARRY_BYTES = 2048;   // in front of every window buffer: the carried span of a hash range (< 1 KiB)

struct pbsgpu_stream {
    pbsgpu_ctx *ctx;
    pbsgpu_cfg cfg;
    pbsgpu_set *set;
    uint64_t window;        // process when this many bytes are buffered
    uint64_t cap;           // device buffer capacity = window + max
    std::vector<uint8_t *> buf;
    std::vector<char> busy; // referenced by an in-flight window
    int cur;
    uint64_t fill;          // bytes buffered (copies enqueued) in buf[cur]
    uint64_t base_off;      // stream offset of buf[cur][0]
    bool finished, started;
    std::deque<StreamJob> inflight;   // FIFO
    std::vector<pbsgpu_chunk> ready;
    size_t ready_pos;
    std::deque<uint64_t> suggested;   // absolute offsets, strictly increasing, not yet behind a cut
    // pinned staging ring
    uint8_t *ring = nullptr;
    uint64_t slot_bytes = 0;
    cudaEvent_t slot_done[RING_SLOTS] = {};
    bool slot_used[RING_SLOTS] = {};
    int slot_next = 0, slot_reserved = -1;
    cudaEvent_t copied = nullptr;     // after the most recent H2D copy into the current window
    // DataBlobs of new chunks
    int blob_mode = PBSGPU_BLOB_NONE;
    std::deque<BlobWindow> blobs;
    // encrypt mode (pbsgpu_stream_crypt): keyed digests, encrypted blobs with one IV per blob
    const pbsgpu_crypt *crypt = nullptr;
    bool iv_seeded = false;
    uint8_t iv_seed[32];
    uint64_t n_blobs = 0;             // blobs encoded so far (index of the next blob's IV)
    // XXH3-64 of registered ranges; hr[k] has registration index hr_base + k
    std::deque<HashRange> hr;
    uint64_t hr_base = 0;
    uint64_t hr_work = 0;             // registration index of the first range with bytes still to hash
    uint64_t hr_blk = 0;              // full blocks of that range hashed so far
    uint64_t hr_end = 0;              // end of the last registered range
    cudaStream_t hs = nullptr;        // every window's hash work, in window order
    uint64_t *d_state = nullptr;      // [2][8] chain state of the range that crosses a window end: read from one slot,
    int state_slot = 0;               // written to the other (state_slot is the one to read); swapped per hash launch
};

extern "C" int pbsgpu_stream_open(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, pbsgpu_set *set, pbsgpu_stream **out) {
    if (!ctx || !out) return PBSGPU_EINVAL;
    Guard g(ctx);
    if (!pbsgpu_cfg_ok(cfg)) return fail(ctx, PBSGPU_EINVAL, "invalid pbsgpu_cfg (use pbsgpu_config)");
    if (set && set->ctx != ctx) return fail(ctx, PBSGPU_EINVAL, "set belongs to another context");
    pbsgpu_stream *s = new pbsgpu_stream();
    s->ctx = ctx; s->cfg = *cfg; s->set = set;
    s->window = std::max<uint64_t>(ctx->stream_window, (uint64_t)cfg->max);
    s->cap = 0; s->cur = 0; s->fill = 0; s->base_off = 0;
    s->buf.assign(ctx->stream_nbuf, nullptr); s->busy.assign(ctx->stream_nbuf, 0);
    s->finished = false; s->started = false; s->ready_pos = 0;
    const char *e = getenv("PBSGPU_STREAM_RING_MB");
    s->slot_bytes = (uint64_t)(e && atoi(e) > 0 ? atoi(e) : 32) << 20;
    *out = s;
    return PBSGPU_OK;
}

// a window buffer with the hash carry area in front of it
static uint8_t *buf_get(pbsgpu_ctx *ctx, uint64_t cap) {
    uint8_t *p = (uint8_t *)ctx->dev.get(CARRY_BYTES + cap);
    return p ? p + CARRY_BYTES : nullptr;
}

static int stream_start(pbsgpu_stream *s) {
    pbsgpu_ctx *ctx = s->ctx;
    if (s->started) return PBSGPU_OK;
    s->cap = s->window + s->cfg.max + 256;
    s->buf[0] = buf_get(ctx, s->cap);                 // further buffers are allocated when first needed
    if (!s->buf[0]) return fail(ctx, PBSGPU_ENOMEM, "stream buffer of %llu bytes failed", (unsigned long long)s->cap);
    if (cudaEventCreateWithFlags(&s->copied, cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, PBSGPU_ECUDA, "cudaEventCreate failed"); }
    s->started = true;
    return PBSGPU_OK;
}

static void window_hash_release(pbsgpu_ctx *ctx, WindowHash *wh) {
    if (!wh) return;
    if (wh->done) { cudaEventSynchronize(wh->done); cudaEventDestroy(wh->done); }
    ctx->dev.put(wh->dev); ctx->pin.put(wh->host);
    (void)cudaGetLastError();
    delete wh;
}

// the window's hashes: wait for its hash work and mark its finished ranges
static int collect_hashes(pbsgpu_stream *s, WindowHash *wh) {
    pbsgpu_ctx *ctx = s->ctx;
    const cudaError_t e = cudaEventSynchronize(wh->done);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, PBSGPU_ECUDA, "stream hash: %s", cudaGetErrorString(e)); }
    for (size_t k = 0; k < wh->seq.size(); k++) {
        HashRange &r = s->hr[wh->seq[k] - s->hr_base];
        r.h = wh->h_out[wh->slot[k]]; r.done = true;
    }
    return PBSGPU_OK;
}

// the window's new chunks -- [0, end) of the first, then from end to end (the carry put the first at offset 0) -- as
// DataBlobs into a pinned block of the stream
static int collect_blobs(pbsgpu_stream *s, const pbsgpu_job *j, const uint8_t *buf) {
    pbsgpu_ctx *ctx = s->ctx;
    const uint64_t nch = j->h_counters[CTR_CHUNKS];
    std::vector<uint64_t> off, len, out_off;
    uint64_t prev = 0, bytes = 0;
    for (uint64_t k = 0; k < nch; k++) {
        const uint64_t end = j->h_out[k].end_off;
        if (!(j->h_out[k].flags & PBSGPU_CHUNK_KNOWN)) {
            off.push_back(prev); len.push_back(end - prev); out_off.push_back(bytes);
            bytes += s->crypt ? pbsgpu_blob_size_enc(end - prev) : pbsgpu_blob_size(end - prev);
        }
        prev = end;
    }
    if (off.empty()) return PBSGPU_OK;
    BlobWindow bw{(uint8_t *)ctx->pin.get(bytes), std::move(out_off), std::vector<uint64_t>(off.size()), 0};
    if (!bw.host) return fail(ctx, PBSGPU_ENOMEM, "pinned blob arena of %llu bytes failed", (unsigned long long)bytes);
    const uint32_t nb = (uint32_t)off.size();
    std::vector<uint8_t> iv(s->crypt ? 16ull * nb : 0);
    int rc = s->crypt ? pbsgpu_stream_ivs(ctx, s->iv_seeded ? s->iv_seed : nullptr, s->n_blobs, nb, iv.data()) : PBSGPU_OK;
    if (rc == PBSGPU_OK)
        rc = pbsgpu_blob_encode(ctx, s->crypt, s->blob_mode, iv.data(), buf, off.data(), len.data(), nb, bw.host, bw.off.data(),
                                bw.len.data(), nullptr);
    if (rc) { ctx->pin.put(bw.host); return rc; }
    s->n_blobs += nb;
    s->blobs.push_back(std::move(bw));
    return PBSGPU_OK;
}

// collect finished windows (all of them if block) in order
static int stream_collect(pbsgpu_stream *s, bool block) {
    while (!s->inflight.empty()) {
        StreamJob sj = s->inflight.front();
        if (!block) {
            cudaError_t q = cudaEventQuery(sj.j->ev[EV_END]);
            if (q == cudaErrorNotReady) { (void)cudaGetLastError(); break; }
        }
        int rc = pbsgpu_job_finish(sj.j);
        s->inflight.pop_front();
        if (rc == PBSGPU_OK && sj.wh) rc = collect_hashes(s, sj.wh);
        if (rc == PBSGPU_OK && s->blob_mode != PBSGPU_BLOB_NONE) rc = collect_blobs(s, sj.j, s->buf[sj.buf]);
        window_hash_release(s->ctx, sj.wh);
        s->busy[sj.buf] = 0;                          // the window's bytes are no longer needed
        if (rc != PBSGPU_OK) { pbsgpu_job_release(sj.j); return rc; }
        const uint64_t nch = sj.j->h_counters[CTR_CHUNKS];
        for (uint64_t k = 0; k < nch; k++) {
            pbsgpu_chunk c = sj.j->h_out[k];          // flags already carry the fused probe's result
            c.stream = 0; c.end_off += sj.base_off;
            s->ready.push_back(c);
        }
        pbsgpu_job_release(sj.j);
    }
    return PBSGPU_OK;
}

// K7's piece form over the window's list, on the stream's hash stream behind the window's bytes
static int hash_enqueue(pbsgpu_stream *s, const std::vector<uint64_t> &off, const std::vector<uint64_t> &len,
                        const std::vector<uint64_t> &first, const std::vector<uint64_t> &blo, const std::vector<uint8_t> &fin,
                        WindowHash &&wh, WindowHash **out) {
    pbsgpu_ctx *ctx = s->ctx;
    const uint32_t n = (uint32_t)off.size();
    // one pinned block: off | len | first | blo | fin, then the results; one device block: the same lists, the results,
    // the block sums
    const uint64_t total = first.back(), fin_words = (n + 7) / 8, list_words = 4ull * n + 1 + fin_words;
    const uint64_t s_word = (list_words + n + 1) & ~1ull;   // 16 B aligned block sums
    const void *tab = nullptr;
    if (int rc = pbsgpu_xxh3_table(ctx, &tab)) return rc;
    if (!s->hs) CK(cudaStreamCreateWithFlags(&s->hs, cudaStreamNonBlocking));
    if (!s->d_state && !(s->d_state = (uint64_t *)ctx->dev.get(128))) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    WindowHash *w = new WindowHash(std::move(wh));
    w->host = ctx->pin.get((list_words + n) * 8);
    w->dev = ctx->dev.get((s_word + total * 8) * 8);
    if (!w->host || !w->dev || cudaEventCreateWithFlags(&w->done, cudaEventDisableTiming) != cudaSuccess) {
        (void)cudaGetLastError(); window_hash_release(ctx, w);
        return fail(ctx, PBSGPU_ENOMEM, "stream hash: allocation failed");
    }
    uint64_t *h = (uint64_t *)w->host, *d = (uint64_t *)w->dev;
    memcpy(h, off.data(), n * 8); memcpy(h + n, len.data(), n * 8); memcpy(h + 2 * n, first.data(), (n + 1) * 8);
    memcpy(h + 3 * n + 1, blo.data(), n * 8); memcpy(h + 4 * n + 1, fin.data(), n);
    w->h_out = h + list_words;
    cudaError_t e = cudaStreamWaitEvent(s->hs, s->copied, 0);   // every byte of the window and of its carry is there
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, h, list_words * 8, cudaMemcpyHostToDevice, s->hs);
    if (e == cudaSuccess)
        e = launch_xxh3_pieces(s->buf[s->cur], d, d + n, d + 2 * n, d + 3 * n + 1, (const uint8_t *)(d + 4 * n + 1), n, total,
                               tab, d + s_word, s->d_state + 8 * s->state_slot, s->d_state + 8 * (1 - s->state_slot),
                               d + list_words, s->hs);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h + list_words, d + list_words, n * 8, cudaMemcpyDeviceToHost, s->hs);
    if (e == cudaSuccess) e = cudaEventRecord(w->done, s->hs);
    if (e != cudaSuccess) {
        (void)cudaGetLastError(); window_hash_release(ctx, w);
        return fail(ctx, PBSGPU_ECUDA, "stream hash: %s", cudaGetErrorString(e));
    }
    // the range that goes on (if any) saved its state in the other slot; a window without a launch has no range that
    // goes on other than the carried one, whose state stays where it is
    s->state_slot = 1 - s->state_slot;
    *out = w;
    return PBSGPU_OK;
}

// Enqueue the hash work of the current window, whose consumed part ends `consumed` bytes into buf[cur], and copy the span
// a later window still needs into the carry area of buf[next].  *out = NULL when the window has nothing to hash.
static int stream_hash(pbsgpu_stream *s, uint64_t consumed, int next, WindowHash **out) {
    pbsgpu_ctx *ctx = s->ctx;
    *out = nullptr;
    const uint64_t w0 = s->base_off, w1 = w0 + consumed;
    std::vector<uint64_t> off, len, first(1, 0), blo;
    std::vector<uint8_t> fin;
    WindowHash wh;
    uint64_t keep = w1;          // first byte a later window still needs
    uint64_t q = s->hr_work, blk = s->hr_blk;
    for (; q < s->hr_base + s->hr.size(); q++, blk = 0) {
        const HashRange &r = s->hr[q - s->hr_base];
        if (r.len == 0) continue;                     // a constant, set when registered
        if (r.off >= w1) break;
        const uint64_t nb = r.len > 240 ? (r.len - 1) >> 10 : 0;
        const uint64_t blk1 = std::min(nb, (w1 - r.off) >> 10);   // full blocks that end in this window
        const bool done = r.off + r.len <= w1;
        if (blk1 > blk || done) {
            if (done) { wh.seq.push_back(q); wh.slot.push_back((uint32_t)off.size()); }
            off.push_back(r.off - w0);                // modulo 2^64: the range may have begun in an earlier window
            len.push_back(r.len); blo.push_back(blk); fin.push_back(done);
            first.push_back(first.back() + (blk1 - blk));
        }
        if (!done) {   // crosses the window end: keep its next block, or its tail, or all of a short range
            keep = nb == 0 ? r.off : blk1 < nb ? r.off + (blk1 << 10) : r.off + std::min(nb << 10, r.len - 64);
            blk = blk1;
            break;
        }
    }
    s->hr_work = q; s->hr_blk = q < s->hr_base + s->hr.size() ? blk : 0;
    const uint32_t n = (uint32_t)off.size();
    if (n) {
        int rc = hash_enqueue(s, off, len, first, blo, fin, std::move(wh), out);
        if (rc) return rc;
    }
    const uint64_t carry = w1 - keep;   // stream bytes [keep, w1) go in front of buf[next]
    if (carry) {
        cudaError_t e = cudaMemcpyAsync(s->buf[next] - carry, s->buf[s->cur] + (int64_t)(keep - w0), carry,
                                        cudaMemcpyDeviceToDevice, ctx->copy_stream);
        if (e == cudaSuccess) e = cudaEventRecord(s->copied, ctx->copy_stream);
        if (e != cudaSuccess) {
            (void)cudaGetLastError(); window_hash_release(ctx, *out); *out = nullptr;
            return fail(ctx, PBSGPU_ECUDA, "hash carry copy: %s", cudaGetErrorString(e));
        }
    }
    return PBSGPU_OK;
}

static int stream_process(pbsgpu_stream *s, int eof) {
    pbsgpu_ctx *ctx = s->ctx;
    if (s->fill == 0) return PBSGPU_OK;
    uint64_t off0 = 0, len0 = s->fill;
    // suggested boundaries inside this window, relative to its first byte
    std::vector<uint32_t> fstream;
    std::vector<uint64_t> foff;
    while (!s->suggested.empty() && s->suggested.front() <= s->base_off) s->suggested.pop_front();
    for (uint64_t a : s->suggested) {
        if (a >= s->base_off + s->fill) break;
        fstream.push_back(0); foff.push_back(a - s->base_off);
    }
    pbsgpu_job *j = nullptr;
    int rc = pbsgpu_job_create(ctx, &s->cfg, s->buf[s->cur], &off0, &len0, 1, eof, 1, s->set, fstream.data(), foff.data(), foff.size(), &j);
    if (rc) return rc;
    j->sha_suffix = pbsgpu_crypt_id_key(s->crypt);
    CK(cudaStreamWaitEvent(j->ss, s->copied, 0));       // every byte of the window has arrived before K1 reads it
    // front half now: the cut points decide what has to be carried over.  On a candidate overflow only the front half is
    // rerun: the back half is enqueued once the carry is known.
    for (;;) {
        rc = pbsgpu_job_enqueue_front(j);
        if (rc == PBSGPU_OK) {
            cudaError_t e = cudaMemcpyAsync(j->h_counters, j->d_counters, CTR_HOST * sizeof(unsigned long long), cudaMemcpyDeviceToHost, j->ss);
            if (e == cudaSuccess && !eof) e = cudaMemcpyAsync(j->h_consumed, j->d_consumed, 8, cudaMemcpyDeviceToHost, j->ss);
            if (e == cudaSuccess) e = cudaStreamSynchronize(j->ss);
            if (e != cudaSuccess) { (void)cudaGetLastError(); rc = fail(ctx, PBSGPU_ECUDA, "stream window: %s", cudaGetErrorString(e)); }
        }
        const unsigned long long nc = j->h_counters[CTR_CANDIDATES];
        if (rc == PBSGPU_OK && !pbsgpu_job_overflowed(j, nc)) break;
        if (rc == PBSGPU_OK) rc = pbsgpu_job_prepare_rerun(j, nc);   // dense candidates: redo the front half with room for all
        if (rc != PBSGPU_OK) { pbsgpu_job_release(j); return rc; }
    }
    const uint64_t consumed = eof ? s->fill : j->h_consumed[0];
    const uint64_t rest = s->fill - consumed;
    // next buffer (wait for the oldest window if all are referenced)
    int next = -1;
    const int nb = (int)s->buf.size();
    for (;;) {
        for (int i = 0; i < nb; i++) if (i != s->cur && !s->busy[i]) { next = i; break; }
        if (next >= 0 || s->inflight.empty()) break;
        StreamJob oldest = s->inflight.front();
        cudaEventSynchronize(oldest.j->ev[EV_END]);
        rc = stream_collect(s, false);
        if (rc) { pbsgpu_job_release(j); return rc; }
    }
    if (next < 0) { pbsgpu_job_release(j); return fail(ctx, PBSGPU_ESTATE, "internal: no free stream buffer"); }
    if (!s->buf[next]) {
        s->buf[next] = buf_get(ctx, s->cap);
        if (!s->buf[next]) { pbsgpu_job_release(j); return fail(ctx, PBSGPU_ENOMEM, "stream buffer of %llu bytes failed", (unsigned long long)s->cap); }
    }
    WindowHash *wh = nullptr;
    rc = stream_hash(s, consumed, next, &wh);      // reads buf[cur] behind the window's copies; before the carry below
    if (rc) { pbsgpu_job_release(j); return rc; }
    if (rest) {   // carry: ordered on the copy stream in front of the next window's H2D copies, no host wait
        cudaError_t e = cudaMemcpyAsync(s->buf[next], s->buf[s->cur] + consumed, rest, cudaMemcpyDeviceToDevice, ctx->copy_stream);
        if (e == cudaSuccess) e = cudaEventRecord(s->copied, ctx->copy_stream);
        if (e != cudaSuccess) { (void)cudaGetLastError(); window_hash_release(ctx, wh); pbsgpu_job_release(j); return fail(ctx, PBSGPU_ECUDA, "carry copy: %s", cudaGetErrorString(e)); }
    }
    rc = pbsgpu_job_enqueue_back(j);                          // SHA-256 etc. run while the next window fills
    if (rc != PBSGPU_OK) { window_hash_release(ctx, wh); pbsgpu_job_release(j); return rc; }
    s->busy[s->cur] = 1;
    s->inflight.push_back(StreamJob{j, s->cur, s->base_off, wh});
    s->cur = next; s->fill = rest; s->base_off += consumed;
    return stream_collect(s, false);
}

// enqueue the H2D copy of [p, p+len) into the window(s); p must stay valid until `done` (recorded after the last piece)
static int stream_feed(pbsgpu_stream *s, const uint8_t *p, uint64_t len, cudaEvent_t done) {
    pbsgpu_ctx *ctx = s->ctx;
    while (len) {
        uint64_t room = s->cap - s->fill;
        uint64_t take = std::min(len, std::min(room, s->window > s->fill ? s->window - s->fill : 0));
        if (take == 0) {   // window full: cut what can be cut, keep the undecided tail
            int rc = stream_process(s, 0);
            if (rc) return rc;
            if (s->fill >= s->window) return fail(ctx, PBSGPU_ESTATE, "internal: stream window did not drain");
            continue;
        }
        CK(cudaMemcpyAsync(s->buf[s->cur] + s->fill, p, take, cudaMemcpyHostToDevice, ctx->copy_stream));
        CK(cudaEventRecord(s->copied, ctx->copy_stream));
        s->fill += take; p += take; len -= take;
    }
    if (done) CK(cudaEventRecord(done, ctx->copy_stream));
    if (s->fill >= s->window) return stream_process(s, 0);
    return PBSGPU_OK;
}

static int ring_make(pbsgpu_stream *s) {
    pbsgpu_ctx *ctx = s->ctx;
    if (s->ring) return PBSGPU_OK;
    s->ring = (uint8_t *)ctx->pin.get(s->slot_bytes * RING_SLOTS);
    if (!s->ring) return fail(ctx, PBSGPU_ENOMEM, "pinned staging ring of %llu bytes failed", (unsigned long long)(s->slot_bytes * RING_SLOTS));
    for (int i = 0; i < RING_SLOTS; i++)
        if (cudaEventCreateWithFlags(&s->slot_done[i], cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, PBSGPU_ECUDA, "cudaEventCreate failed"); }
    return PBSGPU_OK;
}

extern "C" uint64_t pbsgpu_stream_slot_bytes(const pbsgpu_stream *s) { return s ? s->slot_bytes : 0; }

// Zero-copy staging: *buf = up to pbsgpu_stream_slot_bytes() of pinned memory owned by the stream; the caller reads its
// io.Reader straight into it and calls commit(n).  Blocks only while all ring slots still wait for their DMA.
extern "C" int pbsgpu_stream_reserve(pbsgpu_stream *s, void **buf) {
    if (!s || !buf) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    if (s->finished) return fail(ctx, PBSGPU_ESTATE, "stream already finished");
    if (s->slot_reserved >= 0) return fail(ctx, PBSGPU_ESTATE, "a reserved slot is still uncommitted");
    int rc = stream_start(s);
    if (rc == PBSGPU_OK) rc = ring_make(s);
    if (rc) return rc;
    const int k = s->slot_next;
    if (s->slot_used[k]) CK(cudaEventSynchronize(s->slot_done[k]));   // its DMA is the oldest in flight
    s->slot_used[k] = false;
    s->slot_reserved = k;
    *buf = s->ring + (uint64_t)k * s->slot_bytes;
    return PBSGPU_OK;
}
extern "C" int pbsgpu_stream_commit(pbsgpu_stream *s, uint64_t len) {
    if (!s) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    if (s->slot_reserved < 0) return fail(ctx, PBSGPU_ESTATE, "commit without reserve");
    if (len > s->slot_bytes) return fail(ctx, PBSGPU_EINVAL, "commit of %llu bytes exceeds the slot (%llu)", (unsigned long long)len, (unsigned long long)s->slot_bytes);
    const int k = s->slot_reserved;
    s->slot_reserved = -1;
    if (len == 0) return PBSGPU_OK;
    s->slot_used[k] = true;
    s->slot_next = (k + 1) % RING_SLOTS;
    return stream_feed(s, s->ring + (uint64_t)k * s->slot_bytes, len, s->slot_done[k]);
}

// write(): pinned caller memory is sent by DMA in place (the call returns when the DMA has read it, so the caller may
// reuse the buffer -- io.Writer semantics); pageable memory goes through the ring slot by slot.
extern "C" int pbsgpu_stream_write(pbsgpu_stream *s, const void *data, uint64_t len) {
    if (!s || (len && !data)) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    if (s->finished) return fail(ctx, PBSGPU_ESTATE, "stream already finished");
    if (s->slot_reserved >= 0) return fail(ctx, PBSGPU_ESTATE, "a reserved slot is still uncommitted");
    int rc = stream_start(s);
    if (rc || len == 0) return rc;
    const uint8_t *p = (const uint8_t *)data;
    if (pbsgpu_is_pinned_ptr(data)) {
        rc = stream_feed(s, p, len, nullptr);
        cudaError_t e = cudaEventSynchronize(s->copied);
        if (rc == PBSGPU_OK && e != cudaSuccess) { (void)cudaGetLastError(); rc = fail(ctx, PBSGPU_ECUDA, "H2D copy: %s", cudaGetErrorString(e)); }
        return rc;
    }
    while (len) {
        void *slot = nullptr;
        rc = pbsgpu_stream_reserve(s, &slot);
        if (rc) return rc;
        const uint64_t take = std::min(len, s->slot_bytes);
        memcpy(slot, p, take);
        rc = pbsgpu_stream_commit(s, take);
        if (rc) return rc;
        p += take; len -= take;
    }
    return PBSGPU_OK;
}

extern "C" uint64_t pbsgpu_stream_position(const pbsgpu_stream *s) { return s ? s->base_off + s->fill : 0; }

extern "C" int pbsgpu_stream_suggest(pbsgpu_stream *s, uint64_t offset) {
    if (!s) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    if (s->finished) return fail(ctx, PBSGPU_ESTATE, "stream already finished");
    if (s->cfg.min < 65) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries need an average chunk size >= 512");
    if (offset < s->base_off + s->fill) return fail(ctx, PBSGPU_EINVAL, "suggested boundary %llu lies behind the write position %llu", (unsigned long long)offset, (unsigned long long)(s->base_off + s->fill));
    if (!s->suggested.empty() && offset <= s->suggested.back()) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries must be strictly increasing");
    if (offset) s->suggested.push_back(offset);   // offset 0 is the stream start: nothing to cut
    return PBSGPU_OK;
}

extern "C" int pbsgpu_stream_blob_mode(pbsgpu_stream *s, int mode) {
    if (!s) return PBSGPU_EINVAL;
    Guard g(s->ctx);
    if ((mode < PBSGPU_BLOB_NONE || mode > PBSGPU_BLOB_LZH) && mode != PBSGPU_BLOB_LZL && mode != PBSGPU_BLOB_LZC)
        return fail(s->ctx, PBSGPU_EINVAL, "unknown blob mode %d", mode);
    if (s->started || s->finished) return fail(s->ctx, PBSGPU_ESTATE, "the blob mode is set before the first byte");
    s->blob_mode = mode;
    return PBSGPU_OK;
}

extern "C" int pbsgpu_stream_crypt(pbsgpu_stream *s, const pbsgpu_crypt *crypt, const uint8_t *iv_seed) {
    if (!s || !crypt) return PBSGPU_EINVAL;
    Guard g(s->ctx);
    if (crypt->ctx != s->ctx) return fail(s->ctx, PBSGPU_EINVAL, "crypt belongs to another context");
    if (s->started || s->finished) return fail(s->ctx, PBSGPU_ESTATE, "encrypt mode is set before the first byte");
    s->crypt = crypt;
    s->iv_seeded = iv_seed != nullptr;
    if (iv_seed) memcpy(s->iv_seed, iv_seed, 32);
    return PBSGPU_OK;
}

extern "C" int pbsgpu_stream_poll_blobs(pbsgpu_stream *s, uint8_t *out, uint64_t out_cap, uint64_t *blob_len, uint64_t cap,
                                        uint64_t *n_out) {
    if (!s || !n_out || (cap && (!out || !blob_len))) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    const uint64_t largest = s->crypt ? pbsgpu_blob_size_enc(s->cfg.max) : pbsgpu_blob_size(s->cfg.max);
    if (out_cap < largest)
        return fail(ctx, PBSGPU_EINVAL, "blob buffer of %llu bytes is smaller than one blob of the largest chunk (%llu)",
                    (unsigned long long)out_cap, (unsigned long long)largest);
    int rc = stream_collect(s, false);
    if (rc) return rc;
    uint64_t k = 0, used = 0;
    while (!s->blobs.empty()) {
        BlobWindow &bw = s->blobs.front();
        for (; bw.next < bw.len.size() && k < cap && used + bw.len[bw.next] <= out_cap; bw.next++, k++) {
            memcpy(out + used, bw.host + bw.off[bw.next], bw.len[bw.next]);
            blob_len[k] = bw.len[bw.next];
            used += bw.len[bw.next];
        }
        if (bw.next < bw.len.size()) break;
        ctx->pin.put(bw.host);
        s->blobs.pop_front();
    }
    *n_out = k;
    return PBSGPU_OK;
}

extern "C" int pbsgpu_stream_hash_range(pbsgpu_stream *s, uint64_t offset, uint64_t len) {
    if (!s) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    if (s->finished) return fail(ctx, PBSGPU_ESTATE, "stream already finished");
    const uint64_t pos = s->base_off + s->fill;
    if (offset < pos) return fail(ctx, PBSGPU_EINVAL, "hash range at %llu lies behind the write position %llu", (unsigned long long)offset, (unsigned long long)pos);
    if (offset < s->hr_end) return fail(ctx, PBSGPU_EINVAL, "hash range at %llu overlaps the previous one (ranges must ascend)", (unsigned long long)offset);
    if (offset + len < offset) return fail(ctx, PBSGPU_EINVAL, "hash range overflows");
    s->hr.push_back(HashRange{offset, len, len ? 0 : xxh3_empty_host(), len == 0});
    s->hr_end = offset + len;
    return PBSGPU_OK;
}

extern "C" int pbsgpu_stream_poll_hashes(pbsgpu_stream *s, uint64_t *out, uint64_t cap, uint64_t *n_out) {
    if (!s || !n_out || (cap && !out)) return PBSGPU_EINVAL;
    Guard g(s->ctx);
    int rc = stream_collect(s, false);
    if (rc) return rc;
    uint64_t k = 0;
    for (; k < cap && !s->hr.empty() && s->hr.front().done; k++) {
        out[k] = s->hr.front().h;
        s->hr.pop_front(); s->hr_base++;
    }
    // an empty range is done when registered, so the work cursor may sit on one that was just handed out
    if (s->hr_work < s->hr_base) { s->hr_work = s->hr_base; s->hr_blk = 0; }
    *n_out = k;
    return PBSGPU_OK;
}

extern "C" int pbsgpu_stream_finish(pbsgpu_stream *s) {
    if (!s) return PBSGPU_EINVAL;
    Guard g(s->ctx);
    if (s->finished) return PBSGPU_OK;
    if (s->slot_reserved >= 0) return fail(s->ctx, PBSGPU_ESTATE, "a reserved slot is still uncommitted");
    if (s->hr_end > s->base_off + s->fill)
        return fail(s->ctx, PBSGPU_EINVAL, "a hash range ends at %llu, past the end of the stream (%llu)",
                    (unsigned long long)s->hr_end, (unsigned long long)(s->base_off + s->fill));
    int rc = stream_process(s, 1);
    if (rc == PBSGPU_OK) rc = stream_collect(s, true);
    if (rc == PBSGPU_OK) s->finished = true;
    return rc;
}

extern "C" int pbsgpu_stream_poll(pbsgpu_stream *s, pbsgpu_chunk *out, uint64_t cap, uint64_t *n_out) {
    if (!s || !n_out || (cap && !out)) return PBSGPU_EINVAL;
    Guard g(s->ctx);
    int rc = stream_collect(s, false);
    if (rc) return rc;
    uint64_t avail = s->ready.size() - s->ready_pos;
    uint64_t k = std::min(avail, cap);
    if (k) memcpy(out, s->ready.data() + s->ready_pos, k * sizeof(pbsgpu_chunk));
    s->ready_pos += k;
    if (s->ready_pos == s->ready.size()) { s->ready.clear(); s->ready_pos = 0; }
    *n_out = k;
    return PBSGPU_OK;
}

extern "C" void pbsgpu_stream_close(pbsgpu_stream *s) {
    if (!s) return;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    cudaStreamSynchronize(ctx->copy_stream);
    for (auto &sj : s->inflight) { window_hash_release(ctx, sj.wh); pbsgpu_job_release(sj.j); }
    for (auto b : s->buf) if (b) ctx->dev.put(b - CARRY_BYTES);
    for (auto &bw : s->blobs) ctx->pin.put(bw.host);
    ctx->dev.put(s->d_state);
    if (s->hs) cudaStreamDestroy(s->hs);
    if (s->ring) ctx->pin.put(s->ring);
    for (auto e : s->slot_done) if (e) cudaEventDestroy(e);
    if (s->copied) cudaEventDestroy(s->copied);
    (void)cudaGetLastError();
    delete s;
}
