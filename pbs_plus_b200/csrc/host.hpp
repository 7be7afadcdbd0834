// pbs_plus_b200/csrc/host.hpp -- host-side state shared by the capi_*.cu translation units (context, pools, jobs).
// Product code: never includes anything under oracle/.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

#include "internal.cuh"

// ---------------------------------------------------------------------------
// small caching allocators (device + pinned host): steady-state batches do not
// hit cudaMalloc / cudaHostAlloc.
// ---------------------------------------------------------------------------
struct Block { void *p; size_t size; bool used; };
struct Pool {
    std::vector<Block> blocks;
    bool pinned = false;
    void *get(size_t need);
    void put(void *p);
    void trim();
    void destroy();
};

constexpr int N_SCAN_STREAMS = 3;
constexpr int N_STREAMS = 32;   // upper bound of stream slots (main + side stream each); beyond 15 slots streams share the 32 HW queues

struct pbsgpu_job;
struct pbsgpu_ctx {
    int device = 0;
    int sm_count = 0;        // SMs the bulk kernels may use (the bulk partition when the GPU is partitioned)
    int sm_total = 0;        // SMs of the device
    cudaDeviceProp prop;
    std::string err;
    std::recursive_mutex mu;
    cudaStream_t streams[N_STREAMS] = {};
    cudaStream_t streams2[N_STREAMS] = {};   // forked side stream per job stream (latency kernel of the hybrid SHA launch)
    cudaStream_t scan_streams[N_SCAN_STREAMS] = {};   // front halves (K1 scan, sort, K2 resolve) in submission order on the scan partition
    int next_scan = 0;
    cudaStream_t copy_stream = nullptr;
    cudaStream_t tail_stream = nullptr;     // K4 (fused probe) + pack + D2H of every job, in submission order
    bool streams_made = false;
    int next_stream = 0;
    int n_slots = 13;        // PBSGPU_SLOTS: slots in use (jobs of one slot queue FIFO); 13 leaves queues for the host framework
    Pool dev, pin;
    bool profiling = false;
    int variant = 0;
    // device copies of the chunker table (re-uploaded when the cfg table changes)
    uint32_t *d_table = nullptr, *d_rot = nullptr;
    void *d_crc_tables = nullptr;   // K6 tables, uploaded on first use
    void *d_xxh_tab = nullptr;      // K7 secret words, uploaded on first use
    void *d_lz_tab = nullptr;       // K9 predefined FSE tables, uploaded on first use
    void *d_zdec_tab = nullptr;     // K13 codes and predefined FSE decoding tables, uploaded on first use
    uint32_t table_cache[256];
    bool table_valid = false;
    cudaEvent_t epoch = nullptr;   // recorded at open; kernel intervals are reported relative to it
    // optional spatial partition (CUDA green contexts): `part_sms` SMs are reserved for the latency
    // kernels of long chunks (streams2), everything else runs on the remaining SMs (streams)
    // Round 2: an optional THIRD partition (PBSGPU_SCAN_SMS, default off) runs only the front halves: K1 is a whole-SM
    // persistent kernel (207 KB of shared memory, 49 k registers per CTA) that cannot be placed on an SM holding SHA
    // blocks.
    int part_sms = 0, bulk_sms = 0, scan_sms = 0;
    CUgreenCtx g_long = nullptr, g_bulk = nullptr, g_scan = nullptr;
    // knobs, read from the environment ONCE PER CONTEXT in pbsgpu_open (never process-wide statics)
    uint64_t stage_bytes = 0;                 // PBSGPU_STAGE_BYTES: host-input staging group size (0 = auto)
    bool scan_lanes = false;                  // PBSGPU_SCAN_LANES
    uint64_t xxh3_cap_blocks = 8ull << 20;    // PBSGPU_XXH3_CAP_BLOCKS
    pbsgpu::ShaTune tune;                     // PBSGPU_SHA_HYBRID / HYBRID_THR_X10 / SPLIT_SPREAD_KB / HYBRID_HEAD_PER_SM
    uint64_t stream_window = 2ull << 30;      // PBSGPU_STREAM_WINDOW
    int stream_nbuf = 12;                     // PBSGPU_STREAM_NBUF: windows in flight per stream
    // long-chunk arena (PBSGPU_BATCH_EARLY_INPUT jobs): one device ring, allocated on first use.  A job reserves
    // total x arena_frac_x16 / 16 + one maximum chunk; the region is reused once the long-chunk kernels of the jobs that
    // held it are done (stream-ordered: the new job's side stream waits on their events, the host never blocks).
    struct ArenaRec { uint64_t lo, hi; cudaEvent_t ev; };
    uint8_t *arena = nullptr;
    uint64_t arena_bytes = 0, arena_cursor = 0;
    uint64_t arena_want = 16ull << 30;        // PBSGPU_ARENA_MB (a fifth of an 80 GB H100; halved until it fits)
    int arena_frac_x16 = 3;                   // PBSGPU_ARENA_FRAC_X16
    bool arena_failed = false;
    std::deque<ArenaRec> arena_recs;
};

int pbsgpu_fail(pbsgpu_ctx *c, int code, const char *fmt, ...);
#define fail pbsgpu_fail
#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e__ = (call);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            (void)cudaGetLastError();                                                                  \
            return fail(ctx, PBSGPU_ECUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
        }                                                                                              \
    } while (0)

// one call at a time per ctx + device binding for this OS thread (goroutines migrate).  The caller's binding is restored
// on exit so a host framework that tracks the current device (torch) is not retargeted behind its back -- but ONLY a
// binding the thread really had: a thread that never touched CUDA reports "device 0" from cudaGetDevice, and restoring
// that with cudaSetDevice(0) would CREATE a primary context on GPU 0 in every process of a multi-GPU job (the
// e2e leg of ranks 1..7 then waits for context creation on rank 0's busy GPU).
// Such a thread is returned to "no context" (cuCtxSetCurrent(NULL)).
struct Guard {
    std::lock_guard<std::recursive_mutex> lk;
    int prev = -1;        // device to restore with cudaSetDevice, or -1
    bool unbind = false;  // the thread had no CUDA context: unbind again on exit
    explicit Guard(pbsgpu_ctx *c);
    ~Guard();
};

bool pbsgpu_is_device_ptr(const void *p);
bool pbsgpu_is_pinned_ptr(const void *p);
bool pbsgpu_cfg_ok(const pbsgpu_cfg *c);

// ---------------------------------------------------------------------------
// Blocking calls (capi_aux.cu, capi_blob.cu, capi_set.cu): the device work is a chain of enqueues on one stream and the
// call returns once it is done.  pbsgpu_finish always synchronises `st`, then maps the chain's first error `e` (or the
// sync's) to PBSGPU_ECUDA "what: ...".  A Blocking keeps that first error (enqueue only while ok()) and the call's pool
// blocks; they go back to the pool in the destructor after one more synchronisation, so on every exit path no kernel
// still uses a block the pool can hand out again.
// ---------------------------------------------------------------------------
int pbsgpu_finish(pbsgpu_ctx *ctx, cudaStream_t st, cudaError_t e, const char *what);
struct Blocking {
    pbsgpu_ctx *ctx;
    cudaStream_t st;
    cudaError_t e = cudaSuccess;
    std::vector<void *> blocks;
    Blocking(pbsgpu_ctx *c, cudaStream_t s) : ctx(c), st(s) {}
    ~Blocking();
    Blocking(const Blocking &) = delete;
    Blocking &operator=(const Blocking &) = delete;
    bool ok() const { return e == cudaSuccess; }
    template <typename T> T *get(uint64_t count) {   // NULL when the pool is exhausted
        void *p = ctx->dev.get(count * sizeof(T));
        if (p) blocks.push_back(p);
        return (T *)p;
    }
    template <typename T> T *upload(const T *h, uint64_t count) {   // get + H2D copy of h[0, count)
        T *d = get<T>(count);
        if (d && ok()) e = cudaMemcpyAsync(d, h, count * sizeof(T), cudaMemcpyHostToDevice, st);
        return d;
    }
    // The caller's ranges [base + off[i], + len[i]) on the device, as one span [base, base + hi) with hi the largest
    // range end: `base` itself when it is device memory or nothing is read (hi == 0: base is never dereferenced), else a
    // block filled by an H2D copy of the span.  ENOMEM / ECUDA when that fails.
    int stage(const void *base, const uint64_t *off, const uint64_t *len, uint32_t n, const uint8_t **dbase);
    int finish(const char *what) { return pbsgpu_finish(ctx, st, e, what); }
};
// A constant table of a kernel (K6, K7, K9, K13): built on the host by `fill` and uploaded to *d on the context's first
// use (freed with the context)
int pbsgpu_upload_table_once(pbsgpu_ctx *ctx, void **d, size_t bytes, void (*fill)(void *));

// ---------------------------------------------------------------------------
// digest set (capi_set.cu)
// ---------------------------------------------------------------------------
struct pbsgpu_set {
    pbsgpu_ctx *ctx;
    pbsgpu::SetTable t;
    uint64_t count;          // digests in the table as far as the host knows (finished operations)
    uint64_t pending_max;    // upper bound of insertions enqueued but not yet reconciled (fused batch probes)
    cudaEvent_t last = nullptr;   // completion of the most recent operation enqueued on the table (any stream)
    bool last_valid = false;
};
// Enqueue "probe (+ insert when do_insert)" of digests on stream `st`, in index order.  The count is *n_dev (a job's chunk
// count, known only on the device) or `cap` when n_dev is NULL; `cap` bounds the launch.  d_hit[cap] (or NULL) receives the
// flags, *d_new is incremented by the number of new digests.  Scratch comes from `scratch` (>= pbsgpu_set_scratch_bytes(cap)).
// `guard`/`guard_max` (optional): the kernels do nothing when *guard > guard_max (the job's candidate buffer overflowed and it
// will be rerun).  An insertion adds `cap` to pending_max until pbsgpu_set_reconcile settles it.
size_t pbsgpu_set_scratch_bytes(uint64_t cap);
int pbsgpu_set_enqueue(pbsgpu_set *s, const uint8_t *d_dig, const unsigned long long *n_dev, uint64_t cap, int do_insert,
                       const unsigned long long *guard, uint64_t guard_max, uint8_t *d_hit, unsigned long long *d_new,
                       void *scratch, cudaStream_t st);
void pbsgpu_set_reconcile(pbsgpu_set *s, uint64_t cap, uint64_t n_new);   // an insertion finished: pending -> count
int pbsgpu_set_process_dev(pbsgpu_set *s, const uint8_t *d_dig, uint64_t n, int do_insert, uint8_t *d_hit);

// ---------------------------------------------------------------------------
// Job: one batch of device-resident streams through K1..K4 on one CUDA stream (capi.cu)
// ---------------------------------------------------------------------------
enum { EV_START, EV_SCAN, EV_SORT, EV_RESOLVE, EV_SHA, EV_END, EV_FORK, EV_JOIN, EV_BULK, EV_BACK, EV_SET, EV_INPUT, EV_COUNT };
// Slots of j->d_counters, zeroed by every front half.  The first CTR_HOST slots are copied back to j->h_counters.
enum { CTR_CANDIDATES, CTR_CHUNKS, CTR_HEAD, CTR_NEW, CTR_HOST, CTR_DEVICE = 8 };
// CREATED: nothing in flight.  FRONT: the front half was (perhaps partly) enqueued.  ENQUEUED: both halves are enqueued,
// EV_END recorded, and a fused probe still has to be settled with the set.  FINISHED: results are on the host.
enum JobState { JOB_CREATED, JOB_FRONT, JOB_ENQUEUED, JOB_FINISHED };

struct pbsgpu_job {
    pbsgpu_ctx *ctx = nullptr;
    cudaStream_t st = nullptr, st2 = nullptr, ss = nullptr;   // back half / long-chunk kernel / front half
    pbsgpu_cfg cfg;
    const uint8_t *base = nullptr;
    std::vector<uint64_t> off, len, tile_first, forced_keys;   // forced_keys: (stream << 40 | offset-1) suggested boundaries
    uint32_t n = 0;
    uint64_t total_bytes = 0, total_tiles = 0, chunk_cap = 0, cand_cap = 0;
    int eof = 1, want_digests = 1, variant = 0;
    bool scan_lanes = false;
    uint32_t fixed_log2 = 0;        // > 0: fixed cuts of 2^fixed_log2 bytes (pbsgpu_batch_opts.fixed_size); no candidates
    pbsgpu_set *set = nullptr;      // fused probe + insert (NULL: none)
    const uint8_t *sha_suffix = nullptr;   // encrypt mode: the crypt's device id_key, K3 computes keyed digests
    // device
    uint64_t *d_off = nullptr, *d_len = nullptr, *d_tile_first = nullptr, *d_cand = nullptr, *d_cand_sorted = nullptr, *d_forced = nullptr;
    unsigned long long *d_counters = nullptr;   // [CTR_DEVICE], indexed by CTR_*
    uint32_t *d_counts = nullptr;
    uint64_t *d_chunk_first = nullptr, *d_consumed = nullptr;
    pbsgpu::ChunkRef *d_chunks = nullptr;
    uint32_t *d_keys = nullptr, *d_keys2 = nullptr, *d_vals = nullptr, *d_vals2 = nullptr;
    uint8_t *d_digests = nullptr, *d_hit = nullptr;
    pbsgpu_chunk *d_out = nullptr;
    void *d_temp = nullptr; size_t temp_bytes = 0;
    void *d_set_scratch = nullptr;
    // long-chunk arena (PBSGPU_BATCH_EARLY_INPUT): the head chunks are copied to ctx->arena + arena_lo, the input buffer is
    // free at EV_INPUT (bulk pass + gather done) instead of EV_END
    bool early = false;          // asked for
    bool early_active = false;   // ... and in effect for the pass enqueued last (hybrid launch + arena available)
    uint64_t arena_lo = 0, arena_len = 0, max_head = 0;
    uint64_t *d_arena_off = nullptr;
    unsigned long long *h_early = nullptr;   // pinned: candidate count as of EV_INPUT (overflow => the input is still needed)
    // pinned host
    unsigned long long *h_counters = nullptr;   // [CTR_HOST]
    pbsgpu_chunk *h_out = nullptr;
    uint64_t *h_consumed = nullptr;
    cudaEvent_t ev[EV_COUNT] = {};
    bool profiling = false;
    JobState state = JOB_CREATED;
    uint32_t reruns = 0;
    pbsgpu_timing timing = {};      // filled by pbsgpu_job_finish
};

int pbsgpu_job_create(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base_dev, const uint64_t *off, const uint64_t *len,
                      uint32_t n, int eof, int want_digests, pbsgpu_set *set, const uint32_t *forced_stream,
                      const uint64_t *forced_off, uint64_t n_forced, pbsgpu_job **out, uint32_t fixed_size = 0);
int pbsgpu_job_enqueue_front(pbsgpu_job *j);
int pbsgpu_job_enqueue_back(pbsgpu_job *j);
int pbsgpu_job_enqueue(pbsgpu_job *j);
// Candidate overflow: the candidate buffer is sized from statistics; a job whose `nc` candidates did not fit is rerun from
// its input.  prepare_rerun is called once the overflowed pass is done: it settles the set for a probe that was
// enqueued, grows the candidate buffers to fit `nc` and counts the rerun; the caller enqueues again.
inline bool pbsgpu_job_overflowed(const pbsgpu_job *j, unsigned long long nc) { return nc > j->cand_cap; }
int pbsgpu_job_prepare_rerun(pbsgpu_job *j, unsigned long long nc);
int pbsgpu_job_finish(pbsgpu_job *j);     // blocks; reruns on candidate overflow; fills j->timing
cudaError_t pbsgpu_job_sync(pbsgpu_job *j);
void pbsgpu_job_release(pbsgpu_job *j);   // waits for what the job still has in flight unless it finished

// K6 (capi_aux.cu) over the device ranges [dbase + off[i], + len[i]) into d_out[n], enqueued on b's stream
int pbsgpu_crc32_enqueue(Blocking &b, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t *d_out);
// K3 (capi_aux.cu) over the device chunks d_refs[0, *d_n) of `base` (n bounds the launch) into d_dig[32 n], keyed with the
// device `suffix` (a crypt's id_key) or plain, enqueued on b's stream with the context's kernel variant
void pbsgpu_sha256_enqueue(Blocking &b, const uint8_t *base, const pbsgpu::ChunkRef *d_refs, const unsigned long long *d_n,
                           uint32_t n, const uint8_t *suffix, uint8_t *d_dig);
// K7 (capi_aux.cu): enqueue-only / collect pair so the fused batch call can put it on a job's stream
struct XxhRun {
    uint64_t *d_off = nullptr, *d_len = nullptr, *d_first = nullptr, *d_out = nullptr, *d_state = nullptr, *d_S = nullptr;
    uint32_t n = 0;
};
int pbsgpu_xxh3_enqueue(pbsgpu_ctx *ctx, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n,
                        cudaStream_t st, XxhRun *r);
int pbsgpu_xxh3_collect(pbsgpu_ctx *ctx, XxhRun *r, uint64_t *hash_out, cudaStream_t st);
void pbsgpu_xxh3_release(pbsgpu_ctx *ctx, XxhRun *r);
int pbsgpu_xxh3_table(pbsgpu_ctx *ctx, const void **tab);   // K7's device table (uploaded on first use)
// DataBlobs (capi_blob.cu) of n ranges with the encoder of `mode` (PBSGPU_BLOB_RAW .. PBSGPU_BLOB_LZH, _LZL, _LZC),
// encrypted with crypt and the IVs iv[16 n] or plain (crypt NULL): blob i at out + out_off[i], out_len[i] bytes (out_len
// and crc_out may be NULL).  Device ranges are encoded in place.  The body of every pbsgpu_blob_encode_batch* call.
int pbsgpu_blob_encode(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, int mode, const uint8_t *iv, const void *base,
                       const uint64_t *off, const uint64_t *len, uint32_t n, uint8_t *out, const uint64_t *out_off,
                       uint64_t *out_len, uint32_t *crc_out);
// The body of pbsgpu_blob_decode_batch (crypt NULL) and _enc (capi_blob.cu), without the argument checks: the archive
// reader decodes its blobs through it into its device cache.
int pbsgpu_blob_decode(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, const void *base, const uint64_t *off, const uint64_t *len,
                       uint32_t n, const uint64_t *chunk_len, const uint8_t *digest, uint8_t *out, const uint64_t *out_off,
                       int32_t *status, uint8_t *digest_out);

// ---------------------------------------------------------------------------
// encrypt mode (capi_crypt.cu): one AES-256 key, its K11 tables on the host (J0, E_K(J0)) and on the device
// ---------------------------------------------------------------------------
struct pbsgpu_crypt {
    pbsgpu_ctx *ctx;
    std::vector<uint8_t> tab;   // pbsgpu::GcmTables, then the 32-byte id_key of keyed digests
    uint8_t *d_tab = nullptr;   // device copy of tab
};
// IVs of blobs first .. first + n - 1 of a stream (16 bytes each): from the OS CSPRNG (getrandom), or, with a 32-byte seed,
// IV_k = SHA-256(seed || k as u64 LE)[0, 16)
int pbsgpu_stream_ivs(pbsgpu_ctx *ctx, const uint8_t *seed, uint64_t first, uint32_t n, uint8_t *iv);
// the crypt's device id_key (K3's keyed suffix), NULL for NULL
inline const uint8_t *pbsgpu_crypt_id_key(const pbsgpu_crypt *c) { return c ? c->d_tab + pbsgpu::gcm_tables_bytes() : nullptr; }

template <typename T> static T pbsgpu_driver_ep(const char *name) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
        (void)cudaGetLastError();
        return nullptr;
    }
    return (T)p;
}
