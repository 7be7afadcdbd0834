/*
 * pbsgpu.h -- C ABI of libpbsgpu.so, the H100-native chunk + digest + probe engine.
 *
 * This is the drop-in boundary for the ONE hot path of pbs-plus that this repo
 * accelerates (SURVEY.md section 8): content-defined chunking (buzhash), per-chunk
 * SHA-256 and the known-digest probe.  The reference (pbs-plus @ 26d6969) is pure
 * Go with CGO disabled and has NO existing FFI for this path; the arithmetic sits
 * behind Go call sites into github.com/pbs-plus/pxar v0.19.2 (reference go.mod:28).
 * Every entry point below names the reference interface it replaces
 * (paths relative to the reference tree).  The cgo binding a maintainer would add
 * is in go/gpuchunk/ and INTEGRATION.md.
 *
 * Conventions: plain C, plain pointers and sizes, no C++/torch types.  Every
 * function returns 0 on success or a negative PBSGPU_E* code; pbsgpu_strerror(ctx)
 * returns the message of the last failure on that context.  No thread-local state:
 * a ctx may be used from any OS thread (goroutines migrate), one call at a time per
 * ctx; different ctxs are independent.  There is NO CPU fallback: if no CUDA device
 * is usable pbsgpu_open fails.
 */
#ifndef PBSGPU_H
#define PBSGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PBSGPU_VERSION 201 /* 0.2.0 */

/* error codes (negative errno values) */
#define PBSGPU_OK 0
#define PBSGPU_EINVAL (-22)  /* bad argument (avg not a power of two, NULL, ...)      */
#define PBSGPU_ENOMEM (-12)  /* host or device allocation failed                      */
#define PBSGPU_ERANGE (-34)  /* caller's output array too small; *n_out = needed      */
#define PBSGPU_ECUDA (-5)    /* CUDA runtime/driver error, see pbsgpu_strerror        */
#define PBSGPU_ENODEV (-19)  /* no usable CUDA device                                 */
#define PBSGPU_ESTATE (-77)  /* call not valid in this state (stream finished, ...)   */

typedef struct pbsgpu_ctx pbsgpu_ctx;
typedef struct pbsgpu_set pbsgpu_set;
typedef struct pbsgpu_job pbsgpu_job;
typedef struct pbsgpu_stream pbsgpu_stream;

/* Chunker parameters.  Replaces buzhash.Config as built by buzhash.NewConfig(4096)
 * at internal/pxarmount/commit.go:302-305 and handed to backupproxy.NewPBSStore at
 * commit.go:296-305.  Derivation = upstream PBS ChunkerImpl::new. */
typedef struct pbsgpu_cfg {
    uint32_t avg;       /* average chunk size, BYTES, power of two, 256 .. 2^29 */
    uint32_t min;       /* avg >> 2                                            */
    uint32_t max;       /* avg << 2                                            */
    uint32_t mask;      /* 2*avg - 1                                           */
    uint32_t break_min; /* mask - 2 : cut iff (h & mask) >= break_min           */
    uint32_t window;    /* 64                                                  */
    uint32_t table[256];
} pbsgpu_cfg;

/* One finished chunk.  Replaces the (end offset, digest) pair the reference's
 * dedup writer appends to the dynamic index for every chunk produced inside
 * transfer.ArchiveWriter.WriteEntryReader (commit.go:720, :858). */
typedef struct pbsgpu_chunk {
    uint32_t stream;    /* index of the input stream in this call                */
    uint32_t flags;     /* PBSGPU_CHUNK_KNOWN: digest already in the set (skip upload) */
    uint64_t end_off;   /* exclusive end offset of the chunk within its stream   */
    uint8_t digest[32]; /* SHA-256 of the raw chunk bytes (CryptModeNone, commit.go:314) */
} pbsgpu_chunk;
#define PBSGPU_CHUNK_KNOWN 1u

typedef struct pbsgpu_devinfo {
    int32_t device;
    int32_t sm_count;
    int32_t cc_major, cc_minor;
    uint64_t total_mem, free_mem;
    char name[64];
} pbsgpu_devinfo;

/* Device-time breakdown of the last finished batch/job, CUDA events on the
 * launching stream (only filled when profiling is on). */
typedef struct pbsgpu_timing {
    float scan_ms, sort_ms, resolve_ms, sha_ms, set_ms, total_ms;
    /* kernel intervals in ms since the context was opened (same CUDA clock for all jobs of
     * a ctx): lets a caller merge overlapping jobs into "time a kernel class was active" */
    float scan_t0, scan_t1, sha_t0, sha_t1;
    float sha_long_ms, sha_bulk_ms; /* hybrid SHA launch: latency kernel (long chunks) / throughput kernel */
    uint64_t bytes, chunks, candidates;
    uint32_t scan_launches, sha_launches, other_launches, reruns;
} pbsgpu_timing;

/* ---- lifecycle -------------------------------------------------------------- */
int pbsgpu_version(void);
int pbsgpu_open(int device, pbsgpu_ctx **out);
void pbsgpu_close(pbsgpu_ctx *ctx);
const char *pbsgpu_strerror(const pbsgpu_ctx *ctx);
int pbsgpu_device_info(pbsgpu_ctx *ctx, pbsgpu_devinfo *out);
int pbsgpu_set_profiling(pbsgpu_ctx *ctx, int on);
/* SM partition in effect (CUDA green contexts; PBSGPU_PARTITION_SMS=n at open): SMs reserved for the
 * long-chunk latency kernels / SMs for everything else; both 0 when the GPU is not partitioned. */
int pbsgpu_partition_info(pbsgpu_ctx *ctx, int *long_sms, int *bulk_sms);
/* SMs that run only the front halves (K1 scan, sort, K2 resolve; PBSGPU_SCAN_SMS=n at open); 0 = they share the bulk SMs. */
int pbsgpu_scan_partition_sms(pbsgpu_ctx *ctx);
/* 0 = tuned kernels (default), 1 = simple cross-check kernels (same results) */
int pbsgpu_set_kernel_variant(pbsgpu_ctx *ctx, int variant);

/* ---- a1: configuration (replaces buzhash.NewConfig, commit.go:302-305) ------- */
/* avg in BYTES; table NULL = built-in default table. */
int pbsgpu_config(uint32_t avg_bytes, const uint32_t *table /*[256] or NULL*/, pbsgpu_cfg *out);
/* The reference passes 4096 = KiB in the upstream client's convention (4 MiB). */
int pbsgpu_config_kib(uint32_t avg_kib, const uint32_t *table, pbsgpu_cfg *out);
const uint32_t *pbsgpu_default_table(void);

/* ---- a2+a3(+a4): batch of independent streams ---------------------------------
 * Replaces, for n files at once, the per-file loop
 *     writer.WriteEntryReader(entry, reader, size)       (commit.go:720, :858)
 * i.e. [pull bytes -> buzhash scan -> cut -> SHA-256(chunk) -> known?].
 * Stream i is bytes [base+off[i], base+off[i]+len[i]).  `base` may be a DEVICE
 * pointer (data already resident in HBM) or a HOST pointer (pageable or pinned;
 * the library stages it through pinned buffers and overlaps H2D with compute).
 * Chunks are returned ordered by (stream, end_off).  If `set` is non-NULL every
 * chunk digest is probed against it in that order (a digest also counts as known
 * if an earlier chunk of the same call had it) and then inserted.
 * Returns PBSGPU_ERANGE with *n_out = required count if cap is too small. */
int pbsgpu_chunk_digest_batch(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                              const uint64_t *len, uint32_t n, pbsgpu_set *set, pbsgpu_chunk *out, uint64_t cap,
                              uint64_t *n_out);

/* Asynchronous form for DEVICE-resident input: submit returns as soon as the
 * kernels are enqueued; several jobs may be in flight (they overlap on the GPU,
 * which hides the sequential tail of the longest chunk's SHA-256).  wait blocks,
 * copies the chunks out and frees the job -- except on PBSGPU_ERANGE, where the job stays
 * valid: call wait again with the capacity reported in *n_out, or pbsgpu_batch_free.
 * (A digest set can be attached with pbsgpu_batch_submit_ex.) */
int pbsgpu_batch_submit(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base_dev, const uint64_t *off,
                        const uint64_t *len, uint32_t n, pbsgpu_job **job);
int pbsgpu_batch_wait(pbsgpu_job *job, pbsgpu_chunk *out, uint64_t cap, uint64_t *n_out, pbsgpu_timing *timing);

/* Extended batch form: everything the calls above take, plus
 *  - SUGGESTED BOUNDARIES (SURVEY.md section 8 a2 caveat): offsets at which the caller would like a cut -- the
 *    starts of the files' PAYLOAD headers when the stream is a pxar v2 payload stream (the bytes the production
 *    chunker sees: 16-byte PAYLOAD header + content per file, concatenated; internal/pxarmount/pxarfs.go:408-411,
 *    writer calls commit.go:720,:858).  Rule (upstream PBS `PayloadChunker`, restated for byte-wise arrival): with
 *    the running chunk starting at `base`, a boundary B with B - base < min is dropped; with min <= B - base <= max
 *    the chunk ends at B unless the hash test cuts earlier; with B - base > max the plain chunker decides and B
 *    stays pending.  Pairs (forced_stream[i], forced_off[i]) sorted by (stream, offset), offsets in (0, len);
 *    needs cfg->min >= 65 (avg >= 512).  Whether pbs-plus/pxar v0.19.2 applies such boundaries is UNVERIFIED;
 *    n_forced = 0 gives the plain chunker.
 *  - a digest set for the asynchronous form too: the probe + insert runs as kernels on the job's stream
 *    (jobs that share a set are ordered in submission order), flags come back with the records.
 *  - stream_xxh3[n] (may be NULL): as pbsgpu_chunk_digest_batch_xxh3 (synchronous form only).
 *  - crypt (may be NULL): keyed digests of encrypt mode (see pbsgpu_crypt_create).
 *  - fixed_size (0 = the chunker): cut every stream at fixed offsets instead -- chunk k covers [k * fixed_size,
 *    min((k + 1) * fixed_size, len)), so only a stream's last chunk is short and an empty stream has no chunk: the chunks
 *    of a fixed index (.fidx, pbsgpu_fidx_build).  A power of two from 4 KiB to 16 MiB (upstream writes 4 MiB); cfg may
 *    then be NULL and n_forced must be 0 (PBSGPU_EINVAL otherwise).  No state crosses a chunk boundary, so an image of any
 *    size can be fed as slices that start at multiples of fixed_size, one call per slice.
 * `size` must be sizeof(pbsgpu_batch_opts) (forward compatibility; the sizes without `fixed_size` and without `crypt`
 * are accepted too and give the fields of those layouts). */
typedef struct pbsgpu_crypt pbsgpu_crypt;
typedef struct pbsgpu_batch_opts {
    uint32_t size, flags;
    pbsgpu_set *set;
    const uint32_t *forced_stream;
    const uint64_t *forced_off;
    uint64_t n_forced;
    uint64_t *stream_xxh3;
    /* encrypt mode (may be NULL): record digests are keyed, SHA-256(chunk || id_key) as upstream
     * CryptConfig::compute_digest, and the set's probe + insert sees the keyed digests.  A caller built against the
     * header without this field passes that layout's size (offsetof(pbsgpu_batch_opts, crypt)) and gets plain digests. */
    const pbsgpu_crypt *crypt;
    uint32_t fixed_size;   /* fixed cuts (see above); callers of the layout without it pass offsetof(pbsgpu_batch_opts, fixed_size) */
} pbsgpu_batch_opts;
int pbsgpu_chunk_digest_batch_ex(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                                 const uint64_t *len, uint32_t n, const pbsgpu_batch_opts *opts, pbsgpu_chunk *out,
                                 uint64_t cap, uint64_t *n_out);
int pbsgpu_batch_submit_ex(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base_dev, const uint64_t *off,
                           const uint64_t *len, uint32_t n, const pbsgpu_batch_opts *opts, pbsgpu_job **job);
/* pbsgpu_batch_opts.flags for pbsgpu_batch_submit_ex.
 * PBSGPU_BATCH_EARLY_INPUT: give the input buffer back BEFORE the job is done.  A batch's results wait for the serial
 * SHA-256 chain of its longest chunk (~0.3 s for a 16 MiB chunk) -- ten times longer than the rest of a 16 GiB batch --
 * and until then the device reads the input.  With this flag the long chunks (about 11 % of the bytes on backup data)
 * are first copied into an arena inside the library (PBSGPU_ARENA_MB, default 32 GiB, halved until it fits; allocated on first use) and hashed
 * from there: pbsgpu_batch_wait_input returns as soon as the bulk pass and that copy are done, the caller may overwrite
 * or free the buffer and submit the next batch into it, and collects the records later with pbsgpu_batch_wait (in
 * submission order when a set is shared).  pbsgpu_batch_input_done is the non-blocking form (1 free, 0 not yet).
 * Results are identical with and without the flag; without it (or when no arena can be allocated) both calls simply
 * report the end of the job. */
#define PBSGPU_BATCH_EARLY_INPUT 1u
int pbsgpu_batch_wait_input(pbsgpu_job *job);
int pbsgpu_batch_input_done(pbsgpu_job *job);
/* Frees a job without collecting it (after a failed wait, or to abandon it); waits for its kernels. */
void pbsgpu_batch_free(pbsgpu_job *job);

/* Boundary scan only (a2): chunk END offsets per stream, no digests.
 * ends: caller array of cap u64; stream_first[i]..stream_first[i+1] index it
 * (stream_first has n+1 entries). */
int pbsgpu_scan_batch(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                      const uint64_t *len, uint32_t n, uint64_t *ends, uint64_t cap, uint64_t *stream_first,
                      uint64_t *n_out);

/* Digest only (a3): SHA-256 of n arbitrary byte ranges; digests = n*32 bytes (host). */
int pbsgpu_sha256_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                        uint8_t *digests);
/* The keyed digests of encrypt mode: SHA-256(range || id_key of crypt) of n byte ranges (upstream
 * CryptConfig::compute_digest). */
int pbsgpu_sha256_keyed_batch(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, const void *base, const uint64_t *off,
                              const uint64_t *len, uint32_t n, uint8_t *digests);

/* ---- streaming form -----------------------------------------------------------
 * Mirrors how the reference feeds ONE io.Reader of known size through the chunker
 * (scan() state carried across reads; commit.go:718-720).  Bytes are buffered on
 * the device; finished chunks become available from poll(); finish() emits the
 * final short chunk.  Results are identical to the batch call on the whole stream
 * no matter how the bytes are split across writes. */
int pbsgpu_stream_open(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, pbsgpu_set *set, pbsgpu_stream **out);
int pbsgpu_stream_write(pbsgpu_stream *s, const void *host_data, uint64_t len);
int pbsgpu_stream_poll(pbsgpu_stream *s, pbsgpu_chunk *out, uint64_t cap, uint64_t *n_out);
int pbsgpu_stream_finish(pbsgpu_stream *s);
void pbsgpu_stream_close(pbsgpu_stream *s);
/* Zero-copy staging for the streaming form: reserve hands out up to pbsgpu_stream_slot_bytes() of PINNED memory owned
 * by the stream (a ring of 8 slots); the caller reads its io.Reader straight into it and commits the byte count, which
 * starts the DMA and returns at once.  reserve blocks only while every slot still waits for its DMA.  write() is
 * reserve + memcpy + commit for pageable memory and a direct DMA for pinned caller memory. */
int pbsgpu_stream_reserve(pbsgpu_stream *s, void **buf);
int pbsgpu_stream_commit(pbsgpu_stream *s, uint64_t len);
uint64_t pbsgpu_stream_slot_bytes(const pbsgpu_stream *s);
/* Suggested boundary at absolute stream offset `offset` (>= bytes written so far, strictly increasing): what the
 * payload-stream writer calls right before it writes a file's PAYLOAD header.  Rule as in pbsgpu_batch_opts. */
int pbsgpu_stream_suggest(pbsgpu_stream *s, uint64_t offset);
/* Bytes written so far (= the payload offset the next entry will get in the mpxar PAYLOAD_REF). */
uint64_t pbsgpu_stream_position(const pbsgpu_stream *s);
/* DataBlobs of the stream's NEW chunks, encoded on the device from the window that holds them.  The mode is set before
 * the first byte (PBSGPU_ESTATE after that) and has the meaning of pbsgpu_blob_encode_batch (RAW), _z, _lz, _lze, _lzh
 * and _lzl (LZL = 7), and _lzc (LZC = 10; the values 6, 8 and 9 are not assigned and are rejected); NONE, the default, encodes nothing.  Blob k belongs to the k-th record without PBSGPU_CHUNK_KNOWN in poll() order, so
 * with a digest set every new digest gets exactly one blob.  A window's blobs become available when its records do, all
 * of them after finish().  poll_blobs copies whole blobs back to back into out[0, out_cap) and their lengths into
 * blob_len[0, cap); out_cap must be at least pbsgpu_blob_size(cfg.max), so every call makes progress. */
enum { PBSGPU_BLOB_NONE = 0, PBSGPU_BLOB_RAW = 1, PBSGPU_BLOB_Z = 2, PBSGPU_BLOB_LZ = 3, PBSGPU_BLOB_LZE = 4,
       PBSGPU_BLOB_LZH = 5, PBSGPU_BLOB_LZL = 7, PBSGPU_BLOB_LZC = 10 };
int pbsgpu_stream_blob_mode(pbsgpu_stream *s, int mode);
int pbsgpu_stream_poll_blobs(pbsgpu_stream *s, uint8_t *out, uint64_t out_cap, uint64_t *blob_len, uint64_t cap,
                             uint64_t *n_out);
/* Encrypt mode for the stream, set before the first byte (PBSGPU_ESTATE after that): its records carry keyed digests
 * (as pbsgpu_batch_opts.crypt) and poll_blobs returns encrypted blobs (pbsgpu_blob_encode_batch_enc) in the stream's
 * blob mode, so out_cap must be at least pbsgpu_blob_size_enc(cfg.max).  The stream draws one IV per blob from the OS
 * CSPRNG (getrandom) when the blob is encoded -- no IV travels through the caller, and none is ever reused.  iv_seed
 * (32 bytes, or NULL) makes the IVs a function of the seed instead, IV_k = SHA-256(iv_seed || k as u64 LE)[0, 16) for the
 * k-th blob of the stream: for tests that compare blobs byte for byte.  A seed must never be used for two streams under
 * one key. */
int pbsgpu_stream_crypt(pbsgpu_stream *s, const pbsgpu_crypt *crypt, const uint8_t *iv_seed);
/* XXH3-64 (seed 0) of the stream bytes [offset, offset + len), registered before they are written: offset at or after
 * pbsgpu_stream_position, ranges ascending and not overlapping (PBSGPU_EINVAL otherwise).  The payload writer registers
 * every file's content.  Each byte is hashed once on the device, in the window that holds it.  poll_hashes returns the
 * hashes in registration order; a hash is available once the window holding the range's last byte has been collected.
 * finish() fails with PBSGPU_EINVAL when a range extends past the end of the stream. */
int pbsgpu_stream_hash_range(pbsgpu_stream *s, uint64_t offset, uint64_t len);
int pbsgpu_stream_poll_hashes(pbsgpu_stream *s, uint64_t *out, uint64_t cap, uint64_t *n_out);

/* ---- a4: known-digest set -------------------------------------------------------
 * Replaces the known-chunk bookkeeping of the reference's dedup session:
 * seeded from the previous snapshot (backupproxy.PreviousBackupRef commit.go:286-294,
 * origPayloadIdx commit.go:324-329), "Only new chunks are uploaded"
 * (docs/pxar-mount.md:105).  Exact 32-byte comparison, device-resident table. */
int pbsgpu_set_create(pbsgpu_ctx *ctx, uint64_t capacity_hint, pbsgpu_set **out);
void pbsgpu_set_destroy(pbsgpu_set *set);
/* d32: n*32 bytes, HOST or DEVICE pointer.  hit (HOST, n bytes, may be NULL):
 * insert: 1 = already present before this call or earlier within it (then inserted);
 * probe : 1 = present in the set (plain membership, nothing inserted). */
int pbsgpu_set_insert(pbsgpu_set *set, const uint8_t *d32, uint64_t n, uint8_t *hit);
int pbsgpu_set_probe(pbsgpu_set *set, const uint8_t *d32, uint64_t n, uint8_t *hit);
int pbsgpu_set_count(pbsgpu_set *set, uint64_t *count);
/* Seed from a PBS dynamic index (.didx) image: 4096-byte header + 40-byte
 * {u64 end_le, digest[32]} entries (what origPayloadIdx holds, commit.go:324-329). */
int pbsgpu_set_seed_didx(pbsgpu_set *set, const uint8_t *didx, uint64_t size, uint64_t *n_entries);
/* Seed from a PBS fixed index (.fidx) image, the previous snapshot's index of the same disk image (as the upstream
 * client does for fixed indexes): its digests, after pbsgpu_fidx_parse's checks without the checksum. */
int pbsgpu_set_seed_fidx(pbsgpu_set *set, const uint8_t *fidx, uint64_t bytes, uint64_t *n_entries);

/* ---- e: multi-GPU merge of the digest set (SURVEY.md section 8 e / 8 b) -----------------------------------------
 * One process (or thread) per GPU chunks its own shard of the files; the ONE exchange step is an NCCL all-gather of
 * every rank's new digests over NVLink, after which every rank inserts ALL gathered digests into its replica of the
 * set in global (rank, index) order.  hit[i] (HOST, n bytes, may be NULL) = this rank's digest i was known before the
 * call or occurs earlier in that global order -- so with files sharded in rank order the flags equal a single-GPU run.
 * Collective: every rank of the communicator must call it, in the same order.  d32 HOST or DEVICE, n may be 0.
 * `nccl_comm` is an ncclComm_t the caller owns (libnccl.so.2 is resolved with dlopen at first use; PBSGPU_NCCL_LIB
 * overrides the path); the three helpers below create one for callers without an NCCL binding of their own
 * (the 128-byte unique id travels by whatever channel the ranks share). */
int pbsgpu_set_allgather(pbsgpu_set *set, void *nccl_comm, const uint8_t *d32, uint64_t n, uint8_t *hit);
int pbsgpu_nccl_unique_id(uint8_t id[128]);
int pbsgpu_nccl_comm_create(pbsgpu_ctx *ctx, const uint8_t id[128], int nranks, int rank, void **comm);
void pbsgpu_nccl_comm_destroy(void *comm);

/* ---- f1 ("next" row of SURVEY.md section 8): PBS dynamic index (.didx) images ----------------
 * The (end offset, digest) list of a finished archive lands in `<name>.mpxar.didx` /
 * `<name>.ppxar.didx` (names at commit.go:321-322; parsed via datastore.ParseDynamicIndex,
 * internal/pxar/format.go:163).  Layout restated from upstream PBS (UNVERIFIED against the Go
 * module): 4096-byte header { magic[8] = 1c 91 4e a5 19 ba b3 cd, uuid[16], ctime i64 LE,
 * index_csum[32] = SHA-256 over the entry table, zero padding } followed by n entries
 * { u64 end_le, digest[32] }.  Offsets are cumulative over the records in the order given (the
 * archive stream is the concatenation of the streams).  The checksum is computed on the GPU. */
uint64_t pbsgpu_didx_size(uint64_t n_entries);
int pbsgpu_didx_build(pbsgpu_ctx *ctx, const pbsgpu_chunk *chunks, uint64_t n, const uint8_t uuid[16], int64_t ctime,
                      uint8_t *out, uint64_t cap);
/* ends / digests may be NULL to only count; verify != 0 recomputes index_csum (PBSGPU_EINVAL on mismatch). */
int pbsgpu_didx_parse(pbsgpu_ctx *ctx, const uint8_t *didx, uint64_t size, uint64_t *ends, uint8_t *digests,
                      uint64_t cap, uint64_t *n_entries, int verify);

/* ---- PBS fixed index (.fidx) images: disk images (`<name>.img.fidx`; a VM backup, or proxmox-backup-client backup
 * disk.img:/dev/sdX).  Layout restated from upstream PBS pbs-datastore fixed_index.rs (UNVERIFIED against the Go
 * module): 4096-byte header { magic[8] = 2f 7f 41 ed 91 fd 0f cd, uuid[16], ctime i64 LE, index_csum[32] = SHA-256 over
 * the digest table, size u64 LE (image bytes), chunk_size u64 LE, zero padding } followed by n = ceil(size / chunk_size)
 * digests of 32 bytes; chunk i covers [i * chunk_size, min((i + 1) * chunk_size, size)).  The records of a batch call
 * with pbsgpu_batch_opts.fixed_size = chunk_size over the image give those digests in order. */
uint64_t pbsgpu_fidx_size(uint64_t n_chunks);
/* digests: n x 32 bytes (HOST); n must be ceil(size / chunk_size), chunk_size in [1, 2^32) (PBSGPU_EINVAL otherwise).
 * The checksum is computed on the GPU. */
int pbsgpu_fidx_build(pbsgpu_ctx *ctx, const uint8_t *digests, uint64_t n, uint64_t size, uint64_t chunk_size,
                      const uint8_t uuid[16], int64_t ctime, uint8_t *out, uint64_t cap);
/* size / chunk_size (may be NULL) receive the header's fields, *n_entries the chunk count; digests (may be NULL to only
 * count) receives n x 32 bytes (PBSGPU_ERANGE when cap < n).  PBSGPU_EINVAL for a wrong magic, a chunk_size of 0 or of
 * 2^32 and more, a length other than 4096 + 32 * ceil(size / chunk_size), and with verify != 0 a checksum mismatch
 * (recomputed on the GPU; ctx may be NULL without verify). */
int pbsgpu_fidx_parse(pbsgpu_ctx *ctx, const uint8_t *fidx, uint64_t bytes, uint64_t *size, uint64_t *chunk_size,
                      uint8_t *digests, uint64_t cap, uint64_t *n_entries, int verify);

/* ---- f3 ("next" row): DataBlob checksums for NEW chunks ---------------------------------------
 * A new chunk is uploaded as a PBS DataBlob { magic[8], crc32 LE of the payload, payload } (upstream
 * pbs-datastore data_blob.rs; POST /dynamic_chunk, reference internal/server/backup/log_cleanup.go:19-31).
 * pbsgpu_crc32_batch computes zlib-compatible CRC-32s of n byte ranges (HOST or DEVICE base) on the GPU;
 * pbsgpu_blob_header fills the 12-byte header of an unencrypted, uncompressed blob. */
int pbsgpu_crc32_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                       uint32_t *crc_out);
void pbsgpu_blob_header(uint32_t crc, uint8_t out[12]);
/* Complete uncompressed DataBlobs { magic[8], crc32 LE, payload } of n byte ranges (the NEW chunks of a batch) in one
 * call: blob i is written to out + out_off[i] (HOST memory, 12 + len[i] bytes; pbsgpu_blob_size gives that), the CRCs
 * come from K6, payload bytes are copied from `base` (HOST or DEVICE).  crc_out (may be NULL) also receives the CRCs. */
uint64_t pbsgpu_blob_size(uint64_t payload_len);
int pbsgpu_blob_encode_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                             uint8_t *out, const uint64_t *out_off, uint32_t *crc_out);
/* The same with the COMPRESSED form where it is smaller (upstream `DataBlob::encode` keeps a zstd payload only then):
 * blob i = { compressed-blob magic, crc32 LE of the frame, zstd frame } or the uncompressed blob as above; out_len[i]
 * receives its size (<= pbsgpu_blob_size(len[i]), which is what the caller reserves at out_off[i]).  The frame is a
 * standard zstd frame (RFC 8878) built on the device from RLE_Blocks -- 128 KiB blocks that are one repeated byte, i.e.
 * the zero runs of disk images and sparse files -- and Raw_Blocks; there is NO match / entropy stage, so data without
 * such runs stays uncompressed.  Any zstd decoder reads the result; it is not byte-identical to libzstd's output for the
 * same input (no two zstd encoders are). */
int pbsgpu_blob_encode_batch_z(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                               uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
/* pbsgpu_blob_encode_batch_z with a match stage: every 128 KiB block that is not one repeated byte is a zstd
 * Compressed_Block -- a greedy LZ77 parse inside the block, raw literals and sequences coded with the predefined FSE
 * tables -- when that is smaller than the block, else a Raw_Block.  Same arguments, limits and errors as _z; each blob is
 * at most the size of its _z blob.  The output is a deterministic function of the chunk bytes. */
int pbsgpu_blob_encode_batch_lz(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
/* pbsgpu_blob_encode_batch_lz with zstd's entropy stage: the same parse, and each Compressed_Block is the smaller of the
 * _lz content and one whose LL / OF / ML codes use tables fitted to the block (FSE_Compressed_Mode, or RLE_Mode for a
 * single code) and whose literals are Huffman-coded (values up to 128), one repeated value (RLE) or raw.  Blocks stay
 * independent (no Repeat_Mode, no Treeless literals).  Same arguments, limits and errors as _lz; each blob is at most the
 * size of its _lz blob.  The output is a deterministic function of the chunk bytes. */
int pbsgpu_blob_encode_batch_lze(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                 uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
/* pbsgpu_blob_encode_batch_lze with Huffman-coded literals whatever their largest value: the tree description is the
 * smaller of the direct 4-bit weight form (values up to 128) and the FSE-compressed weight form, so blocks of binary
 * data, whose literals almost always reach above 128, get entropy-coded literals too.  The same parse and sequence
 * tables; each Compressed_Block is the smallest of the _lz content, the _lze content and this one.  Same arguments,
 * limits and errors as _lze; each blob is at most the size of its _lze blob.  The output is a deterministic function
 * of the chunk bytes. */
int pbsgpu_blob_encode_batch_lzh(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                 uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
/* pbsgpu_blob_encode_batch_lzh plus long-distance matches: repeats anywhere earlier in the same chunk (up to 2^24 - 4
 * bytes back), such as copies of a file inside one chunk or repeated pages of an image, which the block-local parse of
 * _lzh cannot see.  Anchors of a content-defined 64-byte hash are paired with the latest earlier anchor of the same
 * hash, verified and extended; the kept matches (>= 64 bytes, no overlap) become long spans of the blocks they cross,
 * and a block with spans is parsed again around them.  Each Compressed_Block is the smaller of the _lzh content and the
 * span parse's (_lzh on ties), and no block refers to another's state, so each blob is at most the size of its _lzh
 * blob.  Same arguments, limits and errors as _lzh.  The output is a deterministic function of the chunk bytes. */
int pbsgpu_blob_encode_batch_lzl(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                 uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
/* pbsgpu_blob_encode_batch_lzh with a stronger match search: the match at a position is the longest among the 16
 * latest earlier positions of the same chunk with the same 4 bytes, up to 2^24 - 4 bytes back (so sources may lie in
 * any earlier block), and the parse is lazy (it may move on up to 2 bytes to a longer match).  The frame, the entropy
 * stage and the block forms are _lzh's; no block refers to another's state.  Blobs of text-like data come out smaller
 * than libzstd level 3's (DESIGN.md K16 has the measurements); the search costs more device time than _lzh's.  Same
 * arguments and errors as _lzh; ranges < 2^32 bytes.  The output is a deterministic function of the chunk bytes. */
int pbsgpu_blob_encode_batch_lzc(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                 uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);

/* ---- f3, read side: decode and verify unencrypted DataBlobs (restore, mount, verify jobs) ------------------------
 * Blob i is [base + off[i], + len[i]) (HOST or DEVICE); its chunk has chunk_len[i] bytes (the difference of consecutive
 * end offsets of the index, pbsgpu_didx_parse).  Per blob, the checks run in this order and the first that fails sets
 * status[i]:
 *   1. the magic: uncompressed or compressed blob (an encrypted magic gives PBSGPU_DEC_ENCRYPTED, any other BAD_MAGIC;
 *      so does a blob shorter than its 12-byte header);
 *   2. the CRC-32 of the payload against the header (BAD_CRC);
 *   3. the decode (BAD_FRAME): an uncompressed payload is the chunk; a compressed one is one or more zstd frames
 *      (RFC 8878), skippable frames allowed between them.  Every form of RFC 8878 3.1.1 is read; rejected are a
 *      non-zero Dictionary_ID, reserved bits or block types, a Window_Descriptor above 2^31 bytes, a block above
 *      Block_Maximum_Size (a Compressed_Block's content must also stay below 128 KiB), a Frame_Content_Size that
 *      differs from the content, an offset beyond the frame's decoded bytes, invalid FSE or Huffman descriptions
 *      (Huffman codes up to 11 bits), bitstreams with bits left over or missing, and trailing bytes;
 *   4. the decoded size == chunk_len[i] (BAD_SIZE; also when the frames would write beyond chunk_len[i]);
 *   5. the XXH64 content checksum of every frame that has one (BAD_CHECKSUM);
 *   6. the SHA-256 of the chunk against digest[i] (BAD_DIGEST), when digest (n x 32 bytes) is not NULL.
 * digest_out (n x 32, may be NULL) receives the SHA-256 of every blob whose status is OK or BAD_DIGEST.
 * out (HOST or DEVICE; NULL = verify only, no decoded byte leaves the device): chunk i goes to out + out_off[i],
 * chunk_len[i] bytes.  It holds the chunk when status[i] is OK or BAD_DIGEST; otherwise its contents are undefined
 * (a DEVICE out may hold a partial decode, a HOST out is left untouched).
 * A corrupt blob never fails the call: it only sets its own status.  Returns PBSGPU_EINVAL for bad arguments (NULL
 * arrays, chunk_len[i] >= 2^32), ENOMEM / ECUDA for the call's own failures, 0 otherwise.  Encrypted blobs are not
 * decrypted here (pbsgpu_blob_decode_batch_enc reads them with their key); BAD_TAG is never returned here. */
enum { PBSGPU_DEC_OK = 0, PBSGPU_DEC_BAD_MAGIC, PBSGPU_DEC_BAD_CRC, PBSGPU_DEC_ENCRYPTED, PBSGPU_DEC_BAD_FRAME,
       PBSGPU_DEC_BAD_SIZE, PBSGPU_DEC_BAD_CHECKSUM, PBSGPU_DEC_BAD_DIGEST };
int pbsgpu_blob_decode_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                             const uint64_t *chunk_len, const uint8_t *digest, uint8_t *out, const uint64_t *out_off,
                             int32_t *status, uint8_t *digest_out);

/* ---- f3, encrypt mode (BackupConfig's CryptMode, commit.go:314): encrypted DataBlobs ------------------------------
 * A crypt handle holds one 32-byte AES-256 key (the caller hands over the raw key bytes; key files are not read here).
 * create expands the key and uploads its tables to the context's device once; destroy zeroes the key material on the
 * host and on the device.  The handle is used with the context it was created on.
 * An encrypted blob is { magic[8], crc32 LE, iv[16], tag[16], ciphertext } (44-byte header; upstream pbs-datastore
 * data_blob.rs / file_formats.rs, restated, UNVERIFIED against the Go module): the payload -- the zstd frame of `mode`'s
 * encoder when that is smaller than the chunk, else the raw chunk -- is encrypted with AES-256-GCM under the key with the
 * blob's 16-byte IV and no AAD, and the CRC covers the ciphertext.  The magic is the encrypted-compressed one
 * (e6 59 1b bf 0b bf d8 0b) for a frame, the encrypted one (7b 67 85 be 22 2d 4c f0) otherwise.
 * IVs: iv holds n x 16 bytes, one per blob, supplied by the caller, so the output is a pure function of the inputs.
 * GCM's security rests on never using one IV twice under one key: draw every IV from a CSPRNG (upstream draws them at
 * random) and never reuse one.  The library never generates or stores IVs.
 * mode: PBSGPU_BLOB_RAW (encrypt every chunk uncompressed) or PBSGPU_BLOB_Z .. PBSGPU_BLOB_LZH, _LZL, _LZC (the
 * compressor whose frame is used when smaller).  Blob i goes to out + out_off[i] (HOST memory), which must hold pbsgpu_blob_size_enc(len[i])
 * bytes; out_len[i] receives its size.  base is HOST or DEVICE; ranges < 2^36 bytes.  crc_out may be NULL. */
/* create also derives the id_key of keyed digests: PBKDF2-HMAC-SHA256(password = key, salt = "_id_key", 10 iterations,
 * 32 bytes), as upstream CryptConfig::new. */
int pbsgpu_crypt_create(pbsgpu_ctx *ctx, const uint8_t key[32], pbsgpu_crypt **out);
void pbsgpu_crypt_destroy(pbsgpu_crypt *crypt);
uint64_t pbsgpu_blob_size_enc(uint64_t payload_len);
int pbsgpu_blob_encode_batch_enc(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, int mode, const void *base, const uint64_t *off,
                                 const uint64_t *len, uint32_t n, const uint8_t *iv, uint8_t *out, const uint64_t *out_off,
                                 uint64_t *out_len, uint32_t *crc_out);
/* Read side of encrypt mode (upstream `DataBlob::decode(Some(crypt_config), Some(digest))`): pbsgpu_blob_decode_batch
 * for a mix of encrypted and unencrypted blobs, with the same arguments, limits and errors, plus `crypt` (required,
 * created on ctx; otherwise PBSGPU_EINVAL).  Per blob the first failing check sets status[i]:
 *   1. the magic: any of the four (BAD_MAGIC otherwise, and for an encrypted blob shorter than its 44-byte header or
 *      a plain one shorter than 12 bytes); PBSGPU_DEC_ENCRYPTED is never returned here;
 *   2. the CRC-32 of [12, len) of a plain blob, [44, len) of an encrypted one (BAD_CRC);
 *   3. the AES-256-GCM tag of an encrypted blob under the key and its IV, no AAD (BAD_TAG; compared in constant time);
 *   4. decode, size and content checksums as for plain blobs: the plaintext of an encrypted-compressed blob is zstd
 *      frames, that of an encrypted blob is the chunk (BAD_FRAME, BAD_SIZE, BAD_CHECKSUM);
 *   5. the digest against digest[i] (BAD_DIGEST): the keyed digest SHA-256(chunk || id_key) for encrypted blobs, the
 *      plain SHA-256 for the others; digest_out receives the same kind.
 * No unauthenticated plaintext leaves the library: decryption writes into a library-owned stage, and for a blob whose
 * status is BAD_MAGIC, BAD_CRC or BAD_TAG no byte of `out` (host or device) is written. */
enum { PBSGPU_DEC_BAD_TAG = PBSGPU_DEC_BAD_DIGEST + 1 };   /* 8: the statuses continue; only the _enc call returns it */
int pbsgpu_blob_decode_batch_enc(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, const void *base, const uint64_t *off,
                                 const uint64_t *len, uint32_t n, const uint64_t *chunk_len, const uint8_t *digest,
                                 uint8_t *out, const uint64_t *out_off, int32_t *status, uint8_t *digest_out);

/* ---- f3, read side: archives (mount and restore read a payload stream through its index) -------------------------
 * A reader maps byte ranges of the archive an index describes to its chunks, decodes and verifies each chunk it is
 * given once (pbsgpu_blob_decode_batch(_enc)'s checks), keeps the verified chunks in a cache in device memory and
 * serves ranges from that cache (reference PxarFS.readFileContent -> SplitArchiveReader.PayloadReaderAt().ReadAt,
 * internal/pxarmount/pxarfs.go:38, :409-412; restore, internal/pxar/format.go:113-132).  The chunk files themselves are
 * read by the caller: plan names the chunks a read needs, read takes their blobs.
 * open: didx is a .didx image, parsed with pbsgpu_didx_parse's rules; its index_csum is verified on the GPU (EINVAL on a
 * mismatch, and on a chunk of 2^32 bytes or more).  crypt: NULL, or a handle created on ctx (EINVAL otherwise);
 * encrypted chunks are then decrypted and their keyed digests checked, as pbsgpu_blob_decode_batch_enc; without it an
 * encrypted blob gets PBSGPU_DEC_ENCRYPTED.  cache_bytes: device memory for verified chunks; 0 = 256 MiB (pxar-mount's
 * --cache-size default); raised to the index's largest chunk; allocated here (ENOMEM otherwise).
 * close: frees the cache; with a crypt the cache is zeroed first.  size: the archive's length (the last end offset).
 * A reader belongs to its ctx: its calls serialise with every other call on the ctx.
 * Ranges: range i is the archive bytes [off[i], off[i] + len[i]).  With PBSGPU_READ_PAYLOAD, off[i] is a file's
 * payload offset and len[i] its size: the 16 bytes at off[i] must be {PXAR_PAYLOAD u64 LE, 16 + len[i] u64 LE} (pxar
 * v2's PAYLOAD header; restated, UNVERIFIED against the Go module) and the range's output is the content at
 * off[i] + 16.  The header may straddle a chunk boundary.  A range that ends past pbsgpu_reader_size makes the whole
 * call EINVAL.  A zero-length plain range touches no chunk and is OK; chunks of length 0 are never touched.
 * plan: the indices of the chunks the ranges touch that the cache does not hold, ascending and without repeats, into
 * chunk[cap]; their digests into digest (k x 32 bytes, may be NULL), so the caller can open .chunks/<hex> directly.
 * *n_out receives the count; PBSGPU_ERANGE when it exceeds cap.
 * read:
 *   1. every chunk named in blob_chunk is first dropped from the cache; repeated or out-of-range entries are EINVAL;
 *   2. blob j is [blob_base + blob_off[j], + blob_len[j]) (HOST or DEVICE), the DataBlob of chunk blob_chunk[j].  It is
 *      decoded with the reader's crypt (or without one) against the chunk's length and digest from the index, and
 *      blob_status[j] (may be NULL) receives its PBSGPU_DEC_* status.  Every verified blob is cached, also one whose
 *      chunk no range touches (prefetch);
 *   3. ranges are served from the chunks still cached plus the chunks this call verified.  status[i] is OK; or, going
 *      through the range's chunks in ascending order, the first failure: the failed blob's status, or
 *      PBSGPU_DEC_MISSING for a chunk that was neither cached nor given; or after those PBSGPU_DEC_BAD_HEADER;
 *   4. out (HOST or DEVICE) receives range i at out + out_off[i]; those len[i] bytes hold the range when status[i] is
 *      OK and are undefined otherwise, but no byte of a chunk that failed a check ever reaches out: only verified
 *      chunks enter the cache, and ranges are copied from the cache alone;
 *   5. a corrupt blob never fails the call.  EINVAL for bad arguments (NULL arrays, unknown flags), ENOMEM / ECUDA for
 *      the call's own failures.
 * Cache: a FIFO ring over cache_bytes with 256-byte aligned slots in insertion order; a hit does not refresh an entry.
 * When one call supplies more blob bytes than the ring holds, the blobs are decoded in groups that fit: the pieces
 * (range x chunk intersections) of chunks that were cached already are copied before the first group is decoded, and
 * each group's pieces right after that group, before the next group can evict it. */
typedef struct pbsgpu_reader pbsgpu_reader;
int pbsgpu_reader_open(pbsgpu_ctx *ctx, const uint8_t *didx, uint64_t size, const pbsgpu_crypt *crypt,
                       uint64_t cache_bytes, pbsgpu_reader **out);
/* A reader over a disk image's fixed index (.fidx, parsed and verified with pbsgpu_fidx_parse's rules): chunk i ends at
 * min((i + 1) * chunk_size, size), and plan, read, size and close behave as for a .didx reader.  An image has no pxar
 * headers: PBSGPU_READ_PAYLOAD on such a reader is PBSGPU_EINVAL. */
int pbsgpu_reader_open_fidx(pbsgpu_ctx *ctx, const uint8_t *fidx, uint64_t bytes, const pbsgpu_crypt *crypt,
                            uint64_t cache_bytes, pbsgpu_reader **out);
void pbsgpu_reader_close(pbsgpu_reader *r);
uint64_t pbsgpu_reader_size(const pbsgpu_reader *r);
#define PBSGPU_READ_PAYLOAD 1u
#define PBSGPU_READ_DEFLATE_LZC 2u   /* pbsgpu_reader_read_deflate only: deflate as pbsgpu_deflate_batch_lzc */
#define PBSGPU_READ_SPARSE 4u        /* pbsgpu_reader_plan of a .fidx reader only: leave out zero chunks */
int pbsgpu_reader_plan(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                       uint64_t *chunk, uint8_t *digest, uint64_t cap, uint64_t *n_out);
int pbsgpu_reader_read(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                       const void *blob_base, const uint64_t *blob_off, const uint64_t *blob_len,
                       const uint64_t *blob_chunk, uint32_t n_blobs,
                       uint8_t *out, const uint64_t *out_off, int32_t *status, int32_t *blob_status);
enum { PBSGPU_DEC_MISSING = PBSGPU_DEC_BAD_TAG + 1,   /* 9: a chunk the range needs was neither cached nor given */
       PBSGPU_DEC_BAD_HEADER };                        /* 10: READ_PAYLOAD and the 16-byte header does not match */

/* ---- f3, read side: sparse image restore ----------------------------------------------------------------------------
 * A thin-provisioned disk image is mostly zeros.  The sparse restore serves its zero chunks without their blobs and
 * hands back only the data bytes of each range with where they go, so a restore into a zero-initialised target (a new
 * file, or a device the caller zeroed, as upstream's skip-zero restore) writes only the data and keeps the image thin.
 * Zero chunk: chunk i of a .fidx reader is a zero chunk when its index digest equals the digest of clen[i] zero bytes:
 * plain SHA-256, or with the reader's crypt the keyed SHA-256(zeros || id_key).  Those digests (chunk_size and the short
 * last chunk) are computed on the GPU on the reader's first sparse call, not at open.  A zero chunk whose start and end
 * lie on 4 KiB block boundaries (or end at the image's end) -- every zero chunk when chunk_size is a multiple of 4096, as
 * upstream's 4 MiB -- is served by its digest: no blob, no decode, no cache slot.  Any other zero chunk shares a block
 * with its neighbours and is read like a data chunk (planned, given, decoded and scanned).  This trusts the index digest, as dedup does (the index checksum was
 * verified at open); a damaged zero-chunk blob in the store is not noticed here -- checking blobs is
 * pbsgpu_blob_decode_batch's job.
 * Holes: image offsets are cut into 4096-byte blocks aligned to the image (block b is [4096 b, 4096 (b + 1))), not to
 * the range.  Within range i, a block's part inside the range is a hole when all of its bytes are zero.  The data
 * extents of the range are the maximal runs of non-hole block parts, as (image offset, length) pairs, ascending.  They
 * depend only on the image bytes and the range: the zero-chunk rule only saves work.
 * pbsgpu_reader_plan with PBSGPU_READ_SPARSE (a .fidx reader only; EINVAL otherwise) leaves out zero chunks; without
 * the flag it is unchanged and names them.  "Zero chunks" below are the ones served by digest.  pbsgpu_reader_read and _read_deflate refuse the flag with EINVAL.
 * pbsgpu_reader_read_sparse: pbsgpu_reader_read's arguments, blob handling, groups, statuses and argument errors, with
 * these differences:
 *  - a .fidx reader only, and flags 0: a .didx reader, or PBSGPU_READ_PAYLOAD, is EINVAL;
 *  - out is HOST memory (a device out is EINVAL) with len[i] bytes reserved at out + out_off[i]; it receives range i's
 *    data bytes packed, in extent order.  No hole byte is copied from the device;
 *  - ext receives (offset, length) u64 pairs, range i's at ext[2 ext_first[i] ..  2 ext_first[i + 1]) (ext_first has
 *    n + 1 entries).  ext_cap (pairs) must be at least sum ceil(B_i / 2), with B_i the number of 4 KiB blocks range i
 *    touches -- the most extents a range can have -- or the call is EINVAL before any work;
 *  - a range whose status is not OK has no extents, and none of its out bytes are written;
 *  - a blob given for a zero chunk is checked and cached like any other, and its blob_status reported; the range's
 *    output does not depend on it.  A range that touches only zero chunks needs no blob and reads no byte of the cache.
 * The data chunks are read into a device stage of their bytes in the call, K17 maps their all-zero block parts there
 * and K14 copies the data extents out. */
int pbsgpu_reader_read_sparse(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                              const void *blob_base, const uint64_t *blob_off, const uint64_t *blob_len,
                              const uint64_t *blob_chunk, uint32_t n_blobs, uint8_t *out, const uint64_t *out_off,
                              uint64_t *ext, uint64_t ext_cap, uint64_t *ext_first, int32_t *status, int32_t *blob_status);

/* ---- f3, read side: sparse file restore ----------------------------------------------------------------------------
 * The restore of a snapshot's files into a directory (reference restoreNormal / restoreFile, internal/pxar/restore.go)
 * reads file contents from a .didx payload archive sparsely, so files with long zero runs are written thin, as
 * upstream's pxar extractor leaves them.  Both calls take one range form on a .didx reader (a .fidx reader is EINVAL):
 * range i is file_off[i], the payload offset of a file's 16-byte PAYLOAD header; file_size[i], its content size; and
 * the content bytes [pos[i], pos[i] + len[i]) with pos + len <= file_size (a file ending past the archive, or a range
 * outside its file, is EINVAL).  A whole file is pos 0, len = size; a large file can be read in pieces.  Only a range
 * at pos 0 reads and checks its file's header (as pbsgpu_reader_read with PBSGPU_READ_PAYLOAD: BAD_HEADER).
 * Zero chunk: a chunk whose length is the index's longest and whose index digest equals the digest of that many zero
 * bytes, plain or keyed with the reader's crypt (computed on the GPU on the first file-sparse call, not at open) --
 * when two or more chunks of that length share a digest.  Otherwise no chunk is a zero chunk: that digest is one serial
 * SHA-256 chain over the longest length, dearer than fetching and decoding the one chunk it could spare.  A
 * window of zero bytes hashes to 0 under any table, so a zero run is cut only at the chunker's maximum: that one length
 * carries almost all zero chunks.  Zero chunks are never planned, fetched, decoded or cached; they need not lie on
 * block boundaries.  This trusts the index digest, as dedup does.
 * Holes: content offsets are cut into 4096-byte blocks aligned to the file's content start (block b is content bytes
 * [4096 b, 4096 (b + 1))).  Within a range, a block's part inside the range is a hole when all of its bytes are zero;
 * extents are (content offset, length) pairs of the maximal runs of the other parts, ascending.  They depend only on
 * the file's bytes and the range: the zero-chunk rule only saves work.
 * pbsgpu_reader_plan_file_sparse: pbsgpu_reader_plan's outputs and errors for these ranges, leaving out zero chunks.
 * pbsgpu_reader_read_file_sparse: pbsgpu_reader_read_sparse's outputs, statuses and errors for these ranges: host out
 * with len[i] bytes reserved at out + out_off[i] for range i's data bytes, packed; ext / ext_first; ext_cap at least
 * sum ceil(B_i / 2), with B_i the blocks range i touches, checked before any work; a failed range has no extents and
 * none of its out bytes are written; a corrupt blob never fails the call.  The data chunks' bytes, with the zeros of
 * the zero chunks in blocks they share with data chunks, are staged on the device, K17 maps their all-zero block
 * parts, and K14 copies the data extents out. */
int pbsgpu_reader_plan_file_sparse(pbsgpu_reader *r, const uint64_t *file_off, const uint64_t *file_size,
                                   const uint64_t *pos, const uint64_t *len, uint32_t n, uint64_t *chunk, uint8_t *digest,
                                   uint64_t cap, uint64_t *n_out);
int pbsgpu_reader_read_file_sparse(pbsgpu_reader *r, const uint64_t *file_off, const uint64_t *file_size,
                                   const uint64_t *pos, const uint64_t *len, uint32_t n, const void *blob_base,
                                   const uint64_t *blob_off, const uint64_t *blob_len, const uint64_t *blob_chunk,
                                   uint32_t n_blobs, uint8_t *out, const uint64_t *out_off, uint64_t *ext,
                                   uint64_t ext_cap, uint64_t *ext_first, int32_t *status, int32_t *blob_status);

/* ---- f3, read side: zip restore ------------------------------------------------------------------------------------
 * Restore as zip (reference internal/pxar/zip.go, RestoreModeZip): files are compressed on the GPU into raw Deflate
 * streams (RFC 1951) and the host writes the zip container around them (APPNOTE 6.3.x, as Go's archive/zip writes it).
 * Deflate format (tests/deflate_ref.py restates it; DESIGN.md K15): a range is cut into 128 KiB segments coded
 * independently (no match reaches an earlier segment), each with K9a's greedy parse at distances <= 32768 and matches
 * <= 258 bytes, as the smallest of: stored blocks of <= 65535 bytes; one fixed-code block; one dynamic-code block
 * (two-queue Huffman, 15-bit codes, 7-bit code-length code) -- stored, then fixed, on ties.  The stream's last block
 * has BFINAL; any other segment ends byte-aligned (a fixed or dynamic block is followed by an empty stored block).
 * The stream of 0 bytes is 03 00.
 * pbsgpu_deflate_bound(len) = len + 15 * ceil(len / 131072) + 2: every stream of len bytes fits (a segment is never
 * larger than its stored form, at most 3 stored blocks of 5 header bytes).
 * pbsgpu_deflate_batch: n raw Deflate streams of [base + off[i], + len[i]) (HOST or DEVICE base) into out + out_off[i]
 * (HOST or DEVICE, pbsgpu_deflate_bound(len[i]) reserved); out_len[i] = its size, crc_out[i] = the CRC-32 of the range
 * (crc_out may be NULL).  more (may be NULL): more[i] != 0 means a later call continues stream i -- no BFINAL, a
 * byte-aligned end, and len[i] must be a multiple of 128 KiB (EINVAL otherwise; a piece of 0 bytes is no bytes).
 * Concatenating the pieces gives exactly the one-call stream.  Scratch is bounded per pass of 4096 segments, so a call
 * of any size works.
 * pbsgpu_deflate_batch_lzc: pbsgpu_deflate_batch's arguments, rules and format (segments, more, forms, bound), with a
 * hash-chain search and lazy parse in each segment instead of the greedy one (tests/deflate_chain_ref.py restates it;
 * DESIGN.md K16d): a match is the longest of the first 32 earlier positions of the segment with the same 3 bytes, at
 * most 32768 back and 258 long (ties to the nearer); the parse may move on
 * up to 2 positions when the next match's gain (4 length - the distance code's extra bits) is larger by more than 4;
 * a segment takes at most 32768 matches.  Smaller streams at a lower rate; passes of 1024 segments, each with about
 * 3.5 GiB of device scratch.
 * pbsgpu_crc32_combine: the CRC-32 of A || B from crc1 = CRC-32(A), crc2 = CRC-32(B) and len2 = |B| (host only). */
uint64_t pbsgpu_deflate_bound(uint64_t len);
int pbsgpu_deflate_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                         const uint8_t *more, uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
int pbsgpu_deflate_batch_lzc(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                             const uint8_t *more, uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out);
uint32_t pbsgpu_crc32_combine(uint32_t crc1, uint32_t crc2, uint64_t len2);
/* The zip container (host only, no ctx).  An entry: its name bytes (a directory's ends in '/'), Unix st_mode, mtime in
 * seconds since the epoch, method (0 stored, 8 deflate), the CRC-32 and the compressed and uncompressed sizes of its
 * content, and the offset of its local header in the archive.
 *  - Entries whose name does not end in '/' (files: method 8; symlinks: method 0, the content is the target) set flag
 *    bit 3: their local header carries zero CRC and sizes, and a data descriptor (signature, CRC, sizes; 8-byte sizes
 *    when either size is >= 0xFFFFFFFF) follows the content.  Directories: method 0, sizes 0, no descriptor.
 *  - "version made by" is Unix; external attributes are st_mode << 16, plus 0x10 for a directory; flag bit 11 is set
 *    when the name is valid UTF-8 and not ASCII; DOS date and time are UTC, clamped to 1980-2107; an extended timestamp
 *    (0x5455) is written when 0 <= mtime < 2^32.
 *  - The central directory's zip64 extra field carries only the fields that overflow (size, compressed size, offset,
 *    in that order); the zip64 end record and locator are written when the entry count (>= 0xFFFF), the directory's
 *    offset or its size (>= 0xFFFFFFFF) overflow.
 * Each call returns the record's size in bytes and writes it to out only when cap is at least that size.
 * pbsgpu_zip_directory: the central directory of entries e[0..n), starting at archive offset `offset`, with its end
 * records. */
typedef struct pbsgpu_zip_entry {
    const uint8_t *name;
    uint32_t name_len;
    uint32_t mode;
    int64_t mtime;
    uint32_t method;
    uint32_t crc;
    uint64_t comp_size, size;
    uint64_t offset;
} pbsgpu_zip_entry;
/* pbsgpu_reader_read_deflate: pbsgpu_reader_read's arguments and rules (plan, groups, statuses, PBSGPU_READ_PAYLOAD header
 * check, argument errors), but each range's output is its raw Deflate stream, as pbsgpu_deflate_batch writes it (more,
 * crc_out as there): out is HOST memory with pbsgpu_deflate_bound(len[i]) reserved at out + out_off[i] (a device out is
 * EINVAL), out_len[i] is the stream's size, and 0 when status[i] is not OK; no byte of a failed range is written.  The
 * ranges are read into a device stage of the call's total range bytes and deflated there: file bytes never cross PCIe
 * uncompressed.  flags may add PBSGPU_READ_DEFLATE_LZC: the streams are then pbsgpu_deflate_batch_lzc's (plan and read
 * refuse that flag with EINVAL). */
int pbsgpu_reader_read_deflate(pbsgpu_reader *r, const uint64_t *off, const uint64_t *len, uint32_t n, uint32_t flags,
                               const uint8_t *more, const void *blob_base, const uint64_t *blob_off, const uint64_t *blob_len,
                               const uint64_t *blob_chunk, uint32_t n_blobs, uint8_t *out, const uint64_t *out_off,
                               uint64_t *out_len, uint32_t *crc_out, int32_t *status, int32_t *blob_status);
uint64_t pbsgpu_zip_local_header(const pbsgpu_zip_entry *e, uint8_t *out, uint64_t cap);
uint64_t pbsgpu_zip_data_descriptor(const pbsgpu_zip_entry *e, uint8_t *out, uint64_t cap);
uint64_t pbsgpu_zip_directory(const pbsgpu_zip_entry *e, uint64_t n, uint64_t offset, uint8_t *out, uint64_t cap);

/* ---- f2 ("next" row): the commit walk's per-file content hash ----------------------------------
 * emitBackedFile tees every new file through `xxh3.New()` and keeps `h.Sum64()` (reference
 * internal/pxarmount/commit.go:717-725); verifyBackedFileHashes later re-reads every file to recompute
 * it (commit.go:957-976).  XXH3-64, seed 0, default secret (github.com/zeebo/xxh3, go.mod; the published
 * xxHash v0.8 algorithm -- tests pin it against libxxhash).
 * pbsgpu_xxh3_batch hashes n byte ranges (HOST or DEVICE base) on the GPU.
 * pbsgpu_chunk_digest_batch_xxh3 is pbsgpu_chunk_digest_batch plus stream_xxh3[n] (may be NULL): the
 * XXH3-64 of every stream computed from the SAME staged bytes the chunker and SHA-256 read, so the
 * batched commit walk needs no second pass over the file on the host. */
int pbsgpu_xxh3_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                      uint64_t *hash_out);
int pbsgpu_chunk_digest_batch_xxh3(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                                   const uint64_t *len, uint32_t n, pbsgpu_set *set, pbsgpu_chunk *out, uint64_t cap,
                                   uint64_t *n_out, uint64_t *stream_xxh3);

/* ---- pinned staging owned by C, filled by the Go side ----------------------------- */
void *pbsgpu_host_alloc(pbsgpu_ctx *ctx, uint64_t bytes);
void pbsgpu_host_free(pbsgpu_ctx *ctx, void *p);

/* ---- measurement aid: synthetic corpus generated on the device ------------------
 * Same integer recipe as oracle/oracle.c:orc_corpus_fill (SURVEY.md section 8d).
 * Writes files [first_file, first_file+n_files), each file_len bytes, at
 * dst_dev + i*stride. */
typedef struct pbsgpu_corpus {
    uint64_t seed, file_len, block_len;
    uint32_t run_blocks, dup_permille, edit_mode, edit_thresh16;
    uint64_t edit_seed;
} pbsgpu_corpus;
int pbsgpu_corpus_fill(pbsgpu_ctx *ctx, const pbsgpu_corpus *c, uint64_t first_file, uint32_t n_files,
                       void *dst_dev, uint64_t stride);

#ifdef __cplusplus
}
#endif
#endif /* PBSGPU_H */
