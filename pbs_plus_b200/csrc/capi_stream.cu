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
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <deque>

#include "host.hpp"

using namespace pbsgpu;

struct StreamJob { pbsgpu_job *j; int buf; uint64_t base_off; };
constexpr int RING_SLOTS = 8;

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

static int stream_start(pbsgpu_stream *s) {
    pbsgpu_ctx *ctx = s->ctx;
    if (s->started) return PBSGPU_OK;
    s->cap = s->window + s->cfg.max + 256;
    s->buf[0] = (uint8_t *)ctx->dev.get(s->cap);      // further buffers are allocated when first needed
    if (!s->buf[0]) return fail(ctx, PBSGPU_ENOMEM, "stream buffer of %llu bytes failed", (unsigned long long)s->cap);
    if (cudaEventCreateWithFlags(&s->copied, cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, PBSGPU_ECUDA, "cudaEventCreate failed"); }
    s->started = true;
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
        s->busy[sj.buf] = 0;
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
        s->buf[next] = (uint8_t *)ctx->dev.get(s->cap);
        if (!s->buf[next]) { pbsgpu_job_release(j); return fail(ctx, PBSGPU_ENOMEM, "stream buffer of %llu bytes failed", (unsigned long long)s->cap); }
    }
    if (rest) {   // carry: ordered on the copy stream in front of the next window's H2D copies, no host wait
        cudaError_t e = cudaMemcpyAsync(s->buf[next], s->buf[s->cur] + consumed, rest, cudaMemcpyDeviceToDevice, ctx->copy_stream);
        if (e == cudaSuccess) e = cudaEventRecord(s->copied, ctx->copy_stream);
        if (e != cudaSuccess) { (void)cudaGetLastError(); pbsgpu_job_release(j); return fail(ctx, PBSGPU_ECUDA, "carry copy: %s", cudaGetErrorString(e)); }
    }
    rc = pbsgpu_job_enqueue_back(j);                          // SHA-256 etc. run while the next window fills
    if (rc != PBSGPU_OK) { pbsgpu_job_release(j); return rc; }
    s->busy[s->cur] = 1;
    s->inflight.push_back(StreamJob{j, s->cur, s->base_off});
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

extern "C" int pbsgpu_stream_finish(pbsgpu_stream *s) {
    if (!s) return PBSGPU_EINVAL;
    Guard g(s->ctx);
    if (s->finished) return PBSGPU_OK;
    if (s->slot_reserved >= 0) return fail(s->ctx, PBSGPU_ESTATE, "a reserved slot is still uncommitted");
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
    for (auto &sj : s->inflight) pbsgpu_job_release(sj.j);
    for (auto b : s->buf) ctx->dev.put(b);
    if (s->ring) ctx->pin.put(s->ring);
    for (auto e : s->slot_done) if (e) cudaEventDestroy(e);
    if (s->copied) cudaEventDestroy(s->copied);
    (void)cudaGetLastError();
    delete s;
}
