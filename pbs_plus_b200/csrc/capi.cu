// pbs_plus_b200/csrc/capi.cu -- C ABI (include/pbsgpu.h): lifecycle, configuration and the batch pipeline.
//
// Host side of the drop-in boundary: what a Go caller reaches through cgo in place of
// buzhash.NewConfig / backupproxy.NewPBSStore / transfer...WriteEntryReader of the
// reference (internal/pxarmount/commit.go:296-329, :720).  Pure C++ over the CUDA
// runtime; no torch types.  There is no CPU fallback anywhere in this file: every data
// path launches the kernels in scan.cu / resolve.cu / sha256.cu / digestset.cu.
// Sibling translation units: capi_set.cu (digest set, NCCL merge), capi_stream.cu (streaming form),
// capi_aux.cu (index images and the blocking byte-range calls: SHA-256, CRC-32, XXH3), capi_blob.cu (DataBlobs) and
// capi_crypt.cu (encrypt mode's key handle).
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <cub/device/device_radix_sort.cuh>

#include "host.hpp"

using namespace pbsgpu;

static const uint32_t DEFAULT_TABLE[256] = {
#include "default_table.inc"
};

// ---------------------------------------------------------------------------
// pools
// ---------------------------------------------------------------------------
void *Pool::get(size_t need) {
    need = (need + 255) & ~(size_t)255;
    if (need == 0) need = 256;
    int best = -1;
    for (size_t i = 0; i < blocks.size(); i++)
        if (!blocks[i].used && blocks[i].size >= need && blocks[i].size <= need * 2 + 4096 &&
            (best < 0 || blocks[i].size < blocks[best].size)) best = (int)i;
    if (best >= 0) { blocks[best].used = true; return blocks[best].p; }
    void *p = nullptr;
    cudaError_t e = pinned ? cudaHostAlloc(&p, need, cudaHostAllocDefault) : cudaMalloc(&p, need);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        trim();   // drop cached free blocks and retry once
        e = pinned ? cudaHostAlloc(&p, need, cudaHostAllocDefault) : cudaMalloc(&p, need);
        if (e != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
    }
    blocks.push_back({p, need, true});
    return p;
}
void Pool::put(void *p) {
    if (!p) return;
    for (auto &b : blocks) if (b.p == p) { b.used = false; return; }
}
void Pool::trim() {
    std::vector<Block> keep;
    for (auto &b : blocks) {
        if (b.used) keep.push_back(b);
        else if (pinned) cudaFreeHost(b.p); else cudaFree(b.p);
    }
    blocks.swap(keep);
}
void Pool::destroy() {
    for (auto &b : blocks) { if (pinned) cudaFreeHost(b.p); else cudaFree(b.p); }
    blocks.clear();
}

int pbsgpu_fail(pbsgpu_ctx *c, int code, const char *fmt, ...) {
    if (c) {
        char buf[512];
        va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
        c->err = buf;
    }
    return code;
}

Guard::Guard(pbsgpu_ctx *c) : lk(c->mu) {
    static auto getcur = pbsgpu_driver_ep<CUresult (*)(CUcontext *)>("cuCtxGetCurrent");
    CUcontext cur = nullptr;
    const bool known = getcur && getcur(&cur) == CUDA_SUCCESS;
    if (known && cur == nullptr) unbind = true;                    // fresh thread: nothing to restore but "no context"
    else if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = -1; }
    if (prev == c->device) prev = -1;
    else cudaSetDevice(c->device);
}
Guard::~Guard() {
    if (unbind) {
        static auto setcur = pbsgpu_driver_ep<CUresult (*)(CUcontext)>("cuCtxSetCurrent");
        if (setcur) setcur(nullptr);
    } else if (prev >= 0) cudaSetDevice(prev);
}

bool pbsgpu_is_device_ptr(const void *p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}
bool pbsgpu_is_pinned_ptr(const void *p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

// ---------------------------------------------------------------------------
extern "C" int pbsgpu_version(void) { return PBSGPU_VERSION; }
extern "C" const uint32_t *pbsgpu_default_table(void) { return DEFAULT_TABLE; }

extern "C" int pbsgpu_config(uint32_t avg, const uint32_t *table, pbsgpu_cfg *out) {
    if (!out || avg < 256u || avg > (1u << 29) || (avg & (avg - 1))) return PBSGPU_EINVAL;
    out->avg = avg; out->min = avg >> 2; out->max = avg << 2;
    out->mask = avg * 2u - 1u; out->break_min = out->mask - 2u; out->window = 64;
    memcpy(out->table, table ? table : DEFAULT_TABLE, sizeof out->table);
    return PBSGPU_OK;
}
extern "C" int pbsgpu_config_kib(uint32_t avg_kib, const uint32_t *table, pbsgpu_cfg *out) {
    if (avg_kib == 0 || avg_kib > (1u << 19)) return PBSGPU_EINVAL;
    return pbsgpu_config(avg_kib << 10, table, out);
}
bool pbsgpu_cfg_ok(const pbsgpu_cfg *c) {
    return c && c->avg >= 256u && c->avg <= (1u << 29) && !(c->avg & (c->avg - 1)) && c->min == c->avg >> 2 &&
           c->max == c->avg << 2 && c->mask == c->avg * 2u - 1u && c->break_min == c->mask - 2u && c->window == 64;
}

// Spatial partition with CUDA green contexts (driver API, resolved at run time so the library does
// not link libcuda): long-chunk latency kernels get `want` SMs of their own, so they are neither
// slowed by co-resident bulk warps nor packed onto a few SMs.  Returns false when the driver does not
// offer it; streams created before a failure are destroyed by ctx_destroy (streams_made stays false).
struct GreenApi {
    CUresult (*devget)(CUdevice *, int);
    CUresult (*getRes)(CUdevice, CUdevResource *, CUdevResourceType);
    CUresult (*split)(CUdevResource *, unsigned *, const CUdevResource *, CUdevResource *, unsigned, unsigned);
    CUresult (*genDesc)(CUdevResourceDesc *, CUdevResource *, unsigned);
    CUresult (*gcreate)(CUgreenCtx *, CUdevResourceDesc, CUdevice, unsigned);
    CUresult (*gstream)(CUstream *, CUgreenCtx, unsigned, int);
    CUresult (*gdestroy)(CUgreenCtx);
    bool ok() const { return devget && getRes && split && genDesc && gcreate && gstream; }
};
static GreenApi green_api() {
    GreenApi g;
    g.devget = pbsgpu_driver_ep<decltype(g.devget)>("cuDeviceGet");
    g.getRes = pbsgpu_driver_ep<decltype(g.getRes)>("cuDeviceGetDevResource");
    g.split = pbsgpu_driver_ep<decltype(g.split)>("cuDevSmResourceSplitByCount");
    g.genDesc = pbsgpu_driver_ep<decltype(g.genDesc)>("cuDevResourceGenerateDesc");
    g.gcreate = pbsgpu_driver_ep<decltype(g.gcreate)>("cuGreenCtxCreate");
    g.gstream = pbsgpu_driver_ep<decltype(g.gstream)>("cuGreenCtxStreamCreate");
    g.gdestroy = pbsgpu_driver_ep<decltype(g.gdestroy)>("cuGreenCtxDestroy");
    return g;
}

// Builds the green contexts + streams for (long, scan, bulk) = (res_long, res_scan (may be empty), res_bulk); nothing
// reaches the context unless everything succeeded.
static bool adopt_partition(pbsgpu_ctx *ctx, const GreenApi &G, CUdevice dev, std::vector<CUdevResource> res_long,
                            std::vector<CUdevResource> res_scan, std::vector<CUdevResource> res_bulk) {
    auto count = [](const std::vector<CUdevResource> &v) { unsigned c = 0; for (auto &r : v) c += r.sm.smCount; return c; };
    if (res_long.empty() || res_bulk.empty() || count(res_long) == 0 || count(res_bulk) == 0) return false;
    const bool three = !res_scan.empty() && count(res_scan) > 0;
    CUdevResourceDesc dA, dB, dC;
    CUgreenCtx gl = nullptr, gb = nullptr, gs = nullptr;
    bool ok = G.genDesc(&dA, res_long.data(), (unsigned)res_long.size()) == CUDA_SUCCESS &&
              G.genDesc(&dB, res_bulk.data(), (unsigned)res_bulk.size()) == CUDA_SUCCESS &&
              (!three || G.genDesc(&dC, res_scan.data(), (unsigned)res_scan.size()) == CUDA_SUCCESS);
    ok = ok && G.gcreate(&gl, dA, dev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS;
    ok = ok && G.gcreate(&gb, dB, dev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS;
    ok = ok && (!three || G.gcreate(&gs, dC, dev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS);
    cudaStream_t a[N_STREAMS] = {}, b[N_STREAMS] = {}, c[N_SCAN_STREAMS] = {};
    for (int i = 0; i < ctx->n_slots && ok; i++) {
        CUstream sa = nullptr, sb = nullptr;
        ok = G.gstream(&sb, gb, CU_STREAM_NON_BLOCKING, 0) == CUDA_SUCCESS;
        if (ok) b[i] = (cudaStream_t)sb;
        ok = ok && G.gstream(&sa, gl, CU_STREAM_NON_BLOCKING, 0) == CUDA_SUCCESS;
        if (ok) a[i] = (cudaStream_t)sa;
    }
    for (int i = 0; i < N_SCAN_STREAMS && ok && three; i++) {
        CUstream sc = nullptr;
        ok = G.gstream(&sc, gs, CU_STREAM_NON_BLOCKING, 0) == CUDA_SUCCESS;
        if (ok) c[i] = (cudaStream_t)sc;
    }
    if (!ok) {
        for (int i = 0; i < N_STREAMS; i++) { if (a[i]) cudaStreamDestroy(a[i]); if (b[i]) cudaStreamDestroy(b[i]); }
        for (int i = 0; i < N_SCAN_STREAMS; i++) if (c[i]) cudaStreamDestroy(c[i]);
        if (G.gdestroy) { if (gl) G.gdestroy(gl); if (gb) G.gdestroy(gb); if (gs) G.gdestroy(gs); }
        (void)cudaGetLastError();
        return false;
    }
    for (int i = 0; i < N_STREAMS; i++) { ctx->streams[i] = b[i]; ctx->streams2[i] = a[i]; }
    for (int i = 0; i < N_SCAN_STREAMS; i++) ctx->scan_streams[i] = c[i];
    ctx->g_long = gl; ctx->g_bulk = gb; ctx->g_scan = gs;
    ctx->part_sms = (int)count(res_long);
    ctx->bulk_sms = (int)count(res_bulk);
    ctx->scan_sms = three ? (int)count(res_scan) : 0;
    ctx->sm_count = ctx->bulk_sms;   // persistent kernels on the bulk streams (CRC-32, ...) size their grid to the bulk partition
    return true;
}

// Spatial partition with CUDA green contexts (driver API resolved at run time so the library does not link libcuda):
// `want` SMs for the long-chunk latency kernels, `want_scan` SMs for the front halves (K1 is a whole-SM persistent
// kernel that cannot be placed on an SM holding SHA blocks), the rest for everything else.  ONE split call cuts the
// device into groups of `unit` SMs (outputs of one split may be combined into one descriptor); if the driver refuses,
// the two-way split of round 1 (long / rest) is tried, and without green contexts the context runs unpartitioned.
static bool make_partition(pbsgpu_ctx *ctx, int want, int want_scan) {
    const GreenApi G = green_api();
    if (!G.ok()) return false;
    cudaFree(0);   // make sure the primary context exists
    CUdevice dev;
    CUdevResource all;
    if (G.devget(&dev, ctx->device) != CUDA_SUCCESS || G.getRes(dev, &all, CU_DEV_RESOURCE_TYPE_SM) != CUDA_SUCCESS) return false;
    const unsigned unit = 8;
    if (want_scan > 0) {
        CUdevResource grp[64], rem;
        unsigned n = 64;
        const CUresult sr = G.split(grp, &n, &all, &rem, 0, unit);
        if (getenv("PBSGPU_DEBUG")) fprintf(stderr, "[pbsgpu] split(all=%u SMs, unit %u) -> rc %d, %u groups of %u, remainder %u\n",
                                            all.sm.smCount, unit, (int)sr, n, n ? grp[0].sm.smCount : 0, rem.sm.smCount);
        if (sr == CUDA_SUCCESS && n >= 3) {
            const unsigned gsz = grp[0].sm.smCount ? grp[0].sm.smCount : unit;
            const unsigned kl = std::max(1u, ((unsigned)want + gsz - 1) / gsz), ks = std::max(1u, ((unsigned)want_scan + gsz - 1) / gsz);
            if (kl + ks < n) {
                std::vector<CUdevResource> L(grp, grp + kl), S(grp + kl, grp + kl + ks), B(grp + kl + ks, grp + n);
                if (rem.sm.smCount > 0) B.push_back(rem);
                if (adopt_partition(ctx, G, dev, L, S, B)) return true;
                if (getenv("PBSGPU_DEBUG")) fprintf(stderr, "[pbsgpu] 3-way partition (%u + %u groups) refused, trying 2-way\n", kl, ks);
            }
        }
        (void)cudaGetLastError();
    }
    CUdevResource grp[1], rest;
    unsigned n = 1;
    if (G.split(grp, &n, &all, &rest, 0, (unsigned)want) != CUDA_SUCCESS || n < 1 || rest.sm.smCount == 0) return false;
    return adopt_partition(ctx, G, dev, {grp[0]}, {}, {rest});
}

static void ctx_destroy(pbsgpu_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < N_STREAMS; i++) {
        if (ctx->streams[i]) cudaStreamDestroy(ctx->streams[i]);
        if (ctx->streams2[i]) cudaStreamDestroy(ctx->streams2[i]);
    }
    for (int i = 0; i < N_SCAN_STREAMS; i++) if (ctx->scan_streams[i]) cudaStreamDestroy(ctx->scan_streams[i]);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->tail_stream) cudaStreamDestroy(ctx->tail_stream);
    if (ctx->d_table) cudaFree(ctx->d_table);
    if (ctx->d_rot) cudaFree(ctx->d_rot);
    if (ctx->d_crc_tables) cudaFree(ctx->d_crc_tables);
    if (ctx->d_xxh_tab) cudaFree(ctx->d_xxh_tab);
    if (ctx->d_lz_tab) cudaFree(ctx->d_lz_tab);
    if (ctx->d_zdec_tab) cudaFree(ctx->d_zdec_tab);
    for (auto &r : ctx->arena_recs) cudaEventDestroy(r.ev);
    ctx->arena_recs.clear();
    if (ctx->arena) cudaFree(ctx->arena);
    if (ctx->epoch) cudaEventDestroy(ctx->epoch);
    if (ctx->g_long || ctx->g_bulk || ctx->g_scan) {
        auto gdestroy = pbsgpu_driver_ep<CUresult (*)(CUgreenCtx)>("cuGreenCtxDestroy");
        if (gdestroy) { if (ctx->g_long) gdestroy(ctx->g_long); if (ctx->g_bulk) gdestroy(ctx->g_bulk); if (ctx->g_scan) gdestroy(ctx->g_scan); }
    }
    ctx->dev.destroy(); ctx->pin.destroy();
    (void)cudaGetLastError();
    delete ctx;
}

static int env_int(const char *name, int dflt) { const char *e = getenv(name); return e ? atoi(e) : dflt; }

extern "C" int pbsgpu_open(int device, pbsgpu_ctx **out) {
    if (!out) return PBSGPU_EINVAL;
    *out = nullptr;
    // Streams that share a hardware work queue serialise (false dependencies); the default is 8 queues.
    // Only effective if the CUDA context has not been created yet -- hosts that initialise CUDA first
    // (e.g. torch) should export CUDA_DEVICE_MAX_CONNECTIONS=32 themselves (bench.py does).  The variable is
    // only set when the host has not chosen a value (PBSGPU_KEEP_ENV=1 leaves the environment alone).
    if (!env_int("PBSGPU_KEEP_ENV", 0)) setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
    int n = 0, prev = -1;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { (void)cudaGetLastError(); return PBSGPU_ENODEV; }
    if (device < 0 || device >= n) return PBSGPU_ENODEV;
    if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = -1; }
    pbsgpu_ctx *ctx = new pbsgpu_ctx();
    ctx->device = device;
    ctx->dev.pinned = false; ctx->pin.pinned = true;
    int rc = PBSGPU_OK;
    do {
        if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&ctx->prop, device) != cudaSuccess) { rc = PBSGPU_ENODEV; break; }
        ctx->sm_count = ctx->sm_total = ctx->prop.multiProcessorCount;
        // knobs: read ONCE PER CONTEXT (a test or a host may change them between two pbsgpu_open calls)
        ctx->stage_bytes = getenv("PBSGPU_STAGE_BYTES") ? strtoull(getenv("PBSGPU_STAGE_BYTES"), nullptr, 0) : 0;
        ctx->variant = env_int("PBSGPU_VARIANT", 0);
        ctx->scan_lanes = env_int("PBSGPU_SCAN_LANES", 0) != 0;
        if (env_int("PBSGPU_XXH3_CAP_BLOCKS", 0) > 0) ctx->xxh3_cap_blocks = (uint64_t)atoll(getenv("PBSGPU_XXH3_CAP_BLOCKS"));
        ctx->tune.hybrid = env_int("PBSGPU_SHA_HYBRID", ctx->tune.hybrid);
        ctx->tune.thr_x10 = env_int("PBSGPU_HYBRID_THR_X10", ctx->tune.thr_x10);
        ctx->tune.spread_kb = env_int("PBSGPU_SPLIT_SPREAD_KB", ctx->tune.spread_kb);
        ctx->tune.head_per_sm = std::max(1, env_int("PBSGPU_HYBRID_HEAD_PER_SM", ctx->tune.head_per_sm));
        ctx->n_slots = std::max(1, std::min(N_STREAMS, env_int("PBSGPU_SLOTS", ctx->n_slots)));
        if (getenv("PBSGPU_STREAM_WINDOW")) ctx->stream_window = strtoull(getenv("PBSGPU_STREAM_WINDOW"), nullptr, 0);
        ctx->stream_nbuf = std::max(2, std::min(32, env_int("PBSGPU_STREAM_NBUF", ctx->stream_nbuf)));
        if (getenv("PBSGPU_ARENA_MB")) ctx->arena_want = strtoull(getenv("PBSGPU_ARENA_MB"), nullptr, 0) << 20;
        ctx->arena_frac_x16 = std::max(1, std::min(16, env_int("PBSGPU_ARENA_FRAC_X16", ctx->arena_frac_x16)));
        // default: 24 SMs reserved for the long-chunk latency kernels (green contexts); 0 disables
        const int want_part = env_int("PBSGPU_PARTITION_SMS", 24);
        // + PBSGPU_SCAN_SMS SMs that run only the front halves (K1 scan / sort / K2); default 0 = scans share the bulk partition
        const int want_scan = env_int("PBSGPU_SCAN_SMS", 0);
        const bool partitioned = want_part > 0 && want_part + 8 <= ctx->sm_count && make_partition(ctx, want_part, want_scan);
        bool ok = true;
        for (int i = 0; i < ctx->n_slots && !partitioned && ok; i++)
            ok = cudaStreamCreateWithFlags(&ctx->streams[i], cudaStreamNonBlocking) == cudaSuccess &&
                 cudaStreamCreateWithFlags(&ctx->streams2[i], cudaStreamNonBlocking) == cudaSuccess;
        if (!ok || cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaStreamCreateWithFlags(&ctx->tail_stream, cudaStreamNonBlocking) != cudaSuccess) { rc = PBSGPU_ECUDA; break; }
        ctx->streams_made = true;
        if (cudaMalloc(&ctx->d_table, 1024) != cudaSuccess || cudaMalloc(&ctx->d_rot, 65536) != cudaSuccess) { rc = PBSGPU_ENOMEM; break; }
        if (cudaEventCreate(&ctx->epoch) != cudaSuccess || cudaEventRecord(ctx->epoch, ctx->streams[0]) != cudaSuccess ||
            cudaEventSynchronize(ctx->epoch) != cudaSuccess) { rc = PBSGPU_ECUDA; break; }
    } while (0);
    if (rc != PBSGPU_OK) { (void)cudaGetLastError(); ctx_destroy(ctx); ctx = nullptr; }
    if (prev >= 0 && prev != device) cudaSetDevice(prev);
    *out = ctx;
    return rc;
}

extern "C" void pbsgpu_close(pbsgpu_ctx *ctx) {
    if (!ctx) return;
    int prev = -1;
    if (cudaGetDevice(&prev) != cudaSuccess) { (void)cudaGetLastError(); prev = -1; }
    const int dev = ctx->device;
    ctx_destroy(ctx);
    if (prev >= 0 && prev != dev) cudaSetDevice(prev);
}

extern "C" const char *pbsgpu_strerror(const pbsgpu_ctx *ctx) {
    if (!ctx) return "pbsgpu: no context (pbsgpu_open failed: no usable CUDA device?)";
    return ctx->err.c_str();
}

extern "C" int pbsgpu_device_info(pbsgpu_ctx *ctx, pbsgpu_devinfo *out) {
    if (!ctx || !out) return PBSGPU_EINVAL;
    Guard g(ctx);
    memset(out, 0, sizeof *out);
    out->device = ctx->device; out->sm_count = ctx->sm_count;
    out->cc_major = ctx->prop.major; out->cc_minor = ctx->prop.minor;
    size_t fr = 0, tot = 0;
    CK(cudaMemGetInfo(&fr, &tot));
    out->free_mem = fr; out->total_mem = tot;
    strncpy(out->name, ctx->prop.name, sizeof out->name - 1);
    return PBSGPU_OK;
}
extern "C" int pbsgpu_partition_info(pbsgpu_ctx *ctx, int *long_sms, int *bulk_sms) {
    if (!ctx) return PBSGPU_EINVAL;
    if (long_sms) *long_sms = ctx->part_sms;
    if (bulk_sms) *bulk_sms = ctx->bulk_sms;
    return PBSGPU_OK;
}
extern "C" int pbsgpu_scan_partition_sms(pbsgpu_ctx *ctx) { return ctx ? ctx->scan_sms : 0; }
extern "C" int pbsgpu_set_profiling(pbsgpu_ctx *ctx, int on) { if (!ctx) return PBSGPU_EINVAL; ctx->profiling = on != 0; return 0; }
extern "C" int pbsgpu_set_kernel_variant(pbsgpu_ctx *ctx, int v) { if (!ctx || v < 0 || v > 1) return PBSGPU_EINVAL; ctx->variant = v; return 0; }

extern "C" void *pbsgpu_host_alloc(pbsgpu_ctx *ctx, uint64_t bytes) {
    if (!ctx) return nullptr;
    Guard g(ctx);
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void pbsgpu_host_free(pbsgpu_ctx *ctx, void *p) { if (ctx && p) { Guard g(ctx); cudaFreeHost(p); } }

static int upload_table(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, cudaStream_t st) {
    if (ctx->table_valid && memcmp(ctx->table_cache, cfg->table, 1024) == 0) return PBSGPU_OK;
    // all streams must be done with the old table before it is replaced
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpyAsync(ctx->d_table, cfg->table, 1024, cudaMemcpyHostToDevice, st));
    CK(launch_build_rot_table(ctx->d_table, ctx->d_rot, st));
    CK(cudaStreamSynchronize(st));
    memcpy(ctx->table_cache, cfg->table, 1024);
    ctx->table_valid = true;
    return PBSGPU_OK;
}

// ---------------------------------------------------------------------------
// Job: one batch of device-resident streams through K1..K4 on one CUDA stream.
// ---------------------------------------------------------------------------
cudaError_t pbsgpu_job_sync(pbsgpu_job *j) {   // everything the job enqueued, on all of its streams
    cudaError_t e = cudaSuccess, r;
    if (j->ss && j->ss != j->st && (r = cudaStreamSynchronize(j->ss)) != cudaSuccess) e = r;
    if (j->st && (r = cudaStreamSynchronize(j->st)) != cudaSuccess) e = r;
    if (j->st2 && (r = cudaStreamSynchronize(j->st2)) != cudaSuccess) e = r;
    if (j->state == JOB_ENQUEUED && (r = cudaEventSynchronize(j->ev[EV_END])) != cudaSuccess) e = r;   // the tail may run on the tail stream
    if (e != cudaSuccess) (void)cudaGetLastError();
    return e;
}

// The job's fused probe (if any) is done: move its insertions from the set's pending bound into its count.
static void job_settle_set(pbsgpu_job *j) {
    if (j->set && j->state == JOB_ENQUEUED) pbsgpu_set_reconcile(j->set, j->chunk_cap, j->h_counters[CTR_NEW]);
}

// A finished job is not synchronised again: its streams are slot streams shared with later jobs.
void pbsgpu_job_release(pbsgpu_job *j) {
    if (!j) return;
    pbsgpu_ctx *c = j->ctx;
    if (j->state == JOB_FRONT || j->state == JOB_ENQUEUED) {   // abandoned, or an enqueue failed midway
        pbsgpu_job_sync(j);
        job_settle_set(j);
    }
    void *devp[] = {j->d_off, j->d_len, j->d_tile_first, j->d_cand, j->d_cand_sorted, j->d_forced, j->d_counters, j->d_counts,
                    j->d_chunk_first, j->d_consumed, j->d_chunks, j->d_keys, j->d_keys2, j->d_vals, j->d_vals2,
                    j->d_digests, j->d_hit, j->d_out, j->d_temp, j->d_set_scratch, j->d_arena_off};
    for (void *p : devp) c->dev.put(p);
    c->pin.put(j->h_counters); c->pin.put(j->h_out); c->pin.put(j->h_consumed); c->pin.put(j->h_early);
    for (cudaEvent_t e : j->ev) if (e) cudaEventDestroy(e);
    delete j;
}

static uint64_t expected_cand_cap(const pbsgpu_cfg &cfg, uint64_t total) {
    // candidates occur with probability 3/(mask+1) per byte on random data
    long double e = (long double)total * 3.0L / ((long double)cfg.mask + 1.0L);
    uint64_t cap = (uint64_t)(e * 4.0L) + 4096;
    return cap;
}

static size_t sort_temp_bytes(const pbsgpu_job *j) {
    size_t t1 = 0, t2 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, t1, (uint64_t *)nullptr, (uint64_t *)nullptr, (int)j->cand_cap);
    if (j->want_digests)
        cub::DeviceRadixSort::SortPairsDescending(nullptr, t2, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                                  (uint32_t *)nullptr, (uint32_t *)nullptr, (int)j->chunk_cap);
    return std::max(t1, t2) + 256;
}

static int job_alloc(pbsgpu_job *j) {
    pbsgpu_ctx *ctx = j->ctx;
    Pool &d = ctx->dev;
    const uint32_t n = j->n;
#define DALLOC(ptr, type, count)                                                           \
    do {                                                                                   \
        ptr = (type *)d.get(sizeof(type) * (size_t)(count));                               \
        if (!ptr) return fail(ctx, PBSGPU_ENOMEM, "device allocation of %zu bytes failed", \
                              sizeof(type) * (size_t)(count));                             \
    } while (0)
    DALLOC(j->d_off, uint64_t, n + 1);
    DALLOC(j->d_len, uint64_t, n + 1);
    DALLOC(j->d_tile_first, uint64_t, n + 2);
    DALLOC(j->d_cand, uint64_t, j->cand_cap);
    DALLOC(j->d_cand_sorted, uint64_t, j->cand_cap);
    if (!j->forced_keys.empty()) DALLOC(j->d_forced, uint64_t, j->forced_keys.size());
    DALLOC(j->d_counters, unsigned long long, CTR_DEVICE);
    DALLOC(j->d_counts, uint32_t, n + 1);
    DALLOC(j->d_chunk_first, uint64_t, n + 2);
    DALLOC(j->d_consumed, uint64_t, n + 1);
    DALLOC(j->d_chunks, ChunkRef, j->chunk_cap + 1);
    DALLOC(j->d_out, pbsgpu_chunk, j->chunk_cap + 1);
    if (j->want_digests) {
        DALLOC(j->d_keys, uint32_t, j->chunk_cap + 1);
        DALLOC(j->d_keys2, uint32_t, j->chunk_cap + 1);
        DALLOC(j->d_vals, uint32_t, j->chunk_cap + 1);
        DALLOC(j->d_vals2, uint32_t, j->chunk_cap + 1);
        DALLOC(j->d_digests, uint8_t, (j->chunk_cap + 1) * 32);
    }
    if (j->set) {
        DALLOC(j->d_hit, uint8_t, j->chunk_cap + 1);
        DALLOC(j->d_set_scratch, uint8_t, pbsgpu_set_scratch_bytes(j->chunk_cap));
    }
    j->temp_bytes = sort_temp_bytes(j);
    DALLOC(j->d_temp, uint8_t, j->temp_bytes);
#undef DALLOC
    j->h_counters = (unsigned long long *)ctx->pin.get(CTR_HOST * sizeof(unsigned long long));
    j->h_out = (pbsgpu_chunk *)ctx->pin.get(sizeof(pbsgpu_chunk) * (j->chunk_cap + 1));
    j->h_consumed = (uint64_t *)ctx->pin.get(sizeof(uint64_t) * (n + 1));
    if (!j->h_counters || !j->h_out || !j->h_consumed) return fail(ctx, PBSGPU_ENOMEM, "pinned host allocation failed");
    memset(j->h_counters, 0, CTR_HOST * sizeof(unsigned long long));
    return PBSGPU_OK;
}

static int job_place(pbsgpu_job *j, pbsgpu_job **out);

// A job with fixed cuts of `fixed_size` bytes (a power of two, checked by the caller): no chunker table, no candidates.
// Its cfg is the chunk size in every field the back half reads: avg = max = fixed_size keeps every chunk below the hybrid
// launch's threshold (thr_x10 / 10 x avg), so the equal-length chunks all take the throughput kernel -- the latency
// kernel only pays for the few chunks far longer than the rest, and fixed chunks have no such tail.
static int job_create_fixed(pbsgpu_ctx *ctx, const void *base_dev, const uint64_t *off, const uint64_t *len, uint32_t n,
                            pbsgpu_set *set, uint64_t n_forced, uint32_t fixed_size, pbsgpu_job **out) {
    if (n >= (1u << 24)) return fail(ctx, PBSGPU_EINVAL, "too many streams in one batch (%u >= 2^24)", n);
    if (set && set->ctx != ctx) return fail(ctx, PBSGPU_EINVAL, "set belongs to another context");
    if (n_forced) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries do not apply to fixed-size chunks");
    pbsgpu_job *j = new pbsgpu_job();
    j->ctx = ctx; j->base = (const uint8_t *)base_dev; j->n = n; j->eof = 1;
    j->want_digests = 1; j->variant = ctx->variant; j->profiling = ctx->profiling; j->set = set;
    memset(&j->cfg, 0, sizeof j->cfg);
    j->cfg.avg = j->cfg.min = j->cfg.max = fixed_size;
    while ((1u << j->fixed_log2) < fixed_size) j->fixed_log2++;
    j->off.assign(off, off + n); j->len.assign(len, len + n);
    uint64_t total = 0, chunks = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (len[i] >= (1ull << KEY_POS_BITS)) { delete j; return fail(ctx, PBSGPU_EINVAL, "stream %u longer than 2^40 bytes", i); }
        total += len[i];
        chunks += (len[i] + fixed_size - 1) >> j->fixed_log2;
    }
    j->total_bytes = total; j->chunk_cap = chunks; j->cand_cap = 0;
    if (chunks >= (1ull << 31)) { delete j; return fail(ctx, PBSGPU_EINVAL, "batch too large (%llu chunks)", (unsigned long long)chunks); }
    return job_place(j, out);
}

int pbsgpu_job_create(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base_dev, const uint64_t *off, const uint64_t *len,
                      uint32_t n, int eof, int want_digests, pbsgpu_set *set, const uint32_t *forced_stream,
                      const uint64_t *forced_off, uint64_t n_forced, pbsgpu_job **out, uint32_t fixed_size) {
    if (fixed_size) return job_create_fixed(ctx, base_dev, off, len, n, set, n_forced, fixed_size, out);
    if (!pbsgpu_cfg_ok(cfg)) return fail(ctx, PBSGPU_EINVAL, "invalid pbsgpu_cfg (use pbsgpu_config)");
    if (n >= (1u << 24)) return fail(ctx, PBSGPU_EINVAL, "too many streams in one batch (%u >= 2^24)", n);
    if (set && set->ctx != ctx) return fail(ctx, PBSGPU_EINVAL, "set belongs to another context");
    if (set && !want_digests) return fail(ctx, PBSGPU_EINVAL, "a digest set needs digests");
    if (n_forced && (!forced_stream || !forced_off)) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries: NULL arrays");
    if (n_forced && cfg->min < 65) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries need an average chunk size >= 512");
    if (n_forced >= (1ull << 30)) return fail(ctx, PBSGPU_EINVAL, "too many suggested boundaries");
    pbsgpu_job *j = new pbsgpu_job();
    j->ctx = ctx; j->cfg = *cfg; j->base = (const uint8_t *)base_dev; j->n = n; j->eof = eof;
    j->want_digests = want_digests; j->variant = ctx->variant; j->profiling = ctx->profiling; j->set = set;
    j->off.assign(off, off + n); j->len.assign(len, len + n);
    const uint64_t tile = j->variant == 1 ? (uint64_t)SIMPLE_SPAN : (uint64_t)WARP_TILE;
    // the lane-contiguous scan reads through a tensor map anchored at `base`: it needs a 128 B aligned base
    j->scan_lanes = j->variant == 0 && ctx->scan_lanes && (((uintptr_t)j->base) & (scan_lanes_align() - 1)) == 0;
    const uint64_t super = scan_lanes_super_bytes(), super_steps = scan_lanes_steps();
    j->tile_first.resize(n + 1);
    uint64_t tiles = 0, total = 0, chunks = 0;
    const uint64_t min_eff = min_effective(cfg->min);
    for (uint32_t i = 0; i < n; i++) {
        if (len[i] >= (1ull << KEY_POS_BITS)) { delete j; return fail(ctx, PBSGPU_EINVAL, "stream %u longer than 2^40 bytes", i); }
        j->tile_first[i] = tiles;
        if (j->scan_lanes) {   // k_scan_lanes: 8 steps per 64 KiB super-tile of a 128 B aligned stream, then plain tiles
            const uint64_t ns = (off[i] & (scan_lanes_align() - 1)) == 0 ? len[i] / super : 0;
            tiles += ns * super_steps + (len[i] - ns * super + tile - 1) / tile;
        } else {
            tiles += (len[i] + tile - 1) / tile;
        }
        total += len[i];
        chunks += len[i] / min_eff + 1;
    }
    // suggested boundaries become candidate keys "cut after byte B-1" next to the hash candidates (resolve.cu applies
    // the same min/max rule to both, which is exactly upstream's PayloadChunker rule for byte-wise arrival)
    j->forced_keys.reserve(n_forced);
    for (uint64_t k = 0; k < n_forced; k++) {
        const uint32_t s = forced_stream[k];
        const uint64_t b = forced_off[k];
        if (s >= n || b == 0 || b >= len[s]) { delete j; return fail(ctx, PBSGPU_EINVAL, "suggested boundary %llu: stream %u offset %llu out of range", (unsigned long long)k, s, (unsigned long long)b); }
        const uint64_t key = ((uint64_t)s << KEY_POS_BITS) | (b - 1);
        if (!j->forced_keys.empty() && key <= j->forced_keys.back()) { delete j; return fail(ctx, PBSGPU_EINVAL, "suggested boundaries not sorted by (stream, offset) at %llu", (unsigned long long)k); }
        j->forced_keys.push_back(key);
    }
    chunks += n_forced;
    j->tile_first[n] = tiles;
    j->total_tiles = tiles; j->total_bytes = total; j->chunk_cap = chunks;
    if (chunks >= (1ull << 31)) { delete j; return fail(ctx, PBSGPU_EINVAL, "batch too large (%llu chunk slots)", (unsigned long long)chunks); }
    j->cand_cap = expected_cand_cap(*cfg, total) + n_forced;
    if (j->cand_cap >= (1ull << 31)) { delete j; return fail(ctx, PBSGPU_EINVAL, "batch too large (candidate buffer)"); }
    return job_place(j, out);
}

// The job's streams, buffers and events; releases the job on failure.
static int job_place(pbsgpu_job *j, pbsgpu_job **out) {
    pbsgpu_ctx *ctx = j->ctx;
    j->st = ctx->streams[ctx->next_stream];
    j->st2 = ctx->streams2[ctx->next_stream];
    ctx->next_stream = (ctx->next_stream + 1) % ctx->n_slots;
    if (ctx->scan_sms > 0) { j->ss = ctx->scan_streams[ctx->next_scan]; ctx->next_scan = (ctx->next_scan + 1) % N_SCAN_STREAMS; }
    else j->ss = j->st;
    int rc = job_alloc(j);
    if (rc) { pbsgpu_job_release(j); return rc; }
    for (cudaEvent_t &e : j->ev)
        if (cudaEventCreateWithFlags(&e, j->profiling ? cudaEventDefault : cudaEventDisableTiming) != cudaSuccess) {
            e = nullptr;
            pbsgpu_job_release(j);
            return fail(ctx, PBSGPU_ECUDA, "cudaEventCreate failed");
        }
    *out = j;
    return PBSGPU_OK;
}

// Long-chunk arena: reserve a region of the ring for job `j` and make `side` (the stream its gather runs on) wait for
// the latency kernels of the jobs that used the region before.  Returns false when no arena can be had
// (the job then runs without early release).
static bool arena_reserve(pbsgpu_job *j, cudaStream_t side) {
    pbsgpu_ctx *ctx = j->ctx;
    if (!ctx->arena && !ctx->arena_failed) {
        uint64_t want = ctx->arena_want;
        while (want >= (256ull << 20)) {
            if (cudaMalloc((void **)&ctx->arena, want) == cudaSuccess) { ctx->arena_bytes = want; break; }
            (void)cudaGetLastError();
            ctx->arena = nullptr;
            want >>= 1;
        }
        if (!ctx->arena) ctx->arena_failed = true;
        if (getenv("PBSGPU_DEBUG")) fprintf(stderr, "pbsgpu: long-chunk arena %llu MiB\n", (unsigned long long)(ctx->arena_bytes >> 20));
    }
    if (!ctx->arena) return false;
    if (!j->d_arena_off) {
        j->max_head = (uint64_t)ctx->tune.head_per_sm * (uint64_t)(ctx->part_sms > 0 ? ctx->part_sms : 24);
        j->d_arena_off = (uint64_t *)ctx->dev.get(sizeof(uint64_t) * (j->max_head + 32));
        j->h_early = (unsigned long long *)ctx->pin.get(sizeof(unsigned long long));
        if (!j->d_arena_off || !j->h_early) return false;
    }
    uint64_t need = j->total_bytes / 16 * (uint64_t)ctx->arena_frac_x16 + (uint64_t)j->cfg.max + 4096;
    need = std::max<uint64_t>(need, 16ull << 20);   // a granule: bounds the number of live records (and their events) for tiny jobs
    need = std::min((need + 255) & ~255ull, ctx->arena_bytes & ~255ull);
    if (ctx->arena_cursor + need > ctx->arena_bytes) ctx->arena_cursor = 0;
    const uint64_t lo = ctx->arena_cursor, hi = lo + need;
    ctx->arena_cursor = hi;
    for (auto it = ctx->arena_recs.begin(); it != ctx->arena_recs.end();) {
        if (it->lo < hi && lo < it->hi) {
            if (cudaStreamWaitEvent(side, it->ev, 0) != cudaSuccess) { (void)cudaGetLastError(); return false; }
            cudaEventDestroy(it->ev);
            it = ctx->arena_recs.erase(it);
        } else ++it;
    }
    cudaEvent_t ev = nullptr;
    if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    ctx->arena_recs.push_back({lo, hi, ev});   // recorded by the caller right after the latency kernel
    j->arena_lo = lo; j->arena_len = need;
    return true;
}

// The hybrid SHA launch pays off when the long-chunk kernels have SMs of their own (partition); without
// a partition their CTAs pin shared memory for ~0.3 s and starve the whole-SM scan CTAs of later batches
// and the pipelined step gets slower.  PBSGPU_SHA_HYBRID=2 forces it on regardless, 0 turns it off.
static bool hybrid_for(const pbsgpu_ctx *ctx) {
    if (ctx->tune.hybrid == 0) return false;
    return ctx->part_sms > 0 || ctx->tune.hybrid == 2;
}

// front half: inputs -> K1 scan -> sort -> K2 resolve (chunk list known on the device afterwards)
int pbsgpu_job_enqueue_front(pbsgpu_job *j) {
    pbsgpu_ctx *ctx = j->ctx;
    cudaStream_t st = j->ss;   // the scan partition's stream (= the job's own stream when the GPU has no scan partition)
    const uint32_t n = j->n;
    j->state = JOB_FRONT;
    if (j->fixed_log2) {   // fixed cuts: one small chain instead of K1 -> sort -> K2
        if (n) {
            CK(cudaMemcpyAsync(j->d_off, j->off.data(), n * 8, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(j->d_len, j->len.data(), n * 8, cudaMemcpyHostToDevice, st));
        }
        CK(cudaMemsetAsync(j->d_counters, 0, CTR_DEVICE * sizeof(unsigned long long), st));
        if (j->profiling) CK(cudaEventRecord(j->ev[EV_START], st));
        CK(cudaEventRecord(j->ev[EV_SCAN], st));
        if (j->profiling) CK(cudaEventRecord(j->ev[EV_SORT], st));
        CK(launch_fixed_refs(j->d_len, n, j->fixed_log2, j->d_counts, j->d_chunk_first, &j->d_counters[CTR_CHUNKS], j->chunk_cap,
                             j->d_chunks, st));
        CK(cudaEventRecord(j->ev[EV_RESOLVE], st));
        return PBSGPU_OK;
    }
    int rc = upload_table(ctx, &j->cfg, st);
    if (rc) return rc;
    if (n) {
        CK(cudaMemcpyAsync(j->d_off, j->off.data(), n * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(j->d_len, j->len.data(), n * 8, cudaMemcpyHostToDevice, st));
    }
    CK(cudaMemcpyAsync(j->d_tile_first, j->tile_first.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st));
    if (j->d_forced) CK(cudaMemcpyAsync(j->d_forced, j->forced_keys.data(), j->forced_keys.size() * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(j->d_counters, 0, CTR_DEVICE * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(j->d_cand, 0xFF, j->cand_cap * 8, st));   // KEY_SENTINEL padding for the sort
    if (j->profiling) CK(cudaEventRecord(j->ev[EV_START], st));
    // K1
    ScanArgs sa;
    sa.base = j->base; sa.off = j->d_off; sa.len = j->d_len; sa.tile_first = j->d_tile_first; sa.n_streams = n;
    sa.total_tiles = j->total_tiles; sa.mask = j->cfg.mask; sa.break_min = j->cfg.break_min; sa.table = ctx->d_table;
    sa.cand = j->d_cand; sa.cand_cap = j->cand_cap; sa.cand_count = &j->d_counters[CTR_CANDIDATES];
    if (j->variant == 1) CK(launch_scan_simple(sa, st));
    else if (j->scan_lanes) {
        uint64_t extent = 0;
        for (uint32_t i = 0; i < n; i++) extent = std::max(extent, j->off[i] + j->len[i]);
        CK(launch_scan_lanes(sa, ctx->d_rot, ctx->scan_sms > 0 ? ctx->scan_sms : ctx->sm_count, extent, st));
    }
    else CK(launch_scan_tuned(sa, ctx->d_rot, ctx->scan_sms > 0 ? ctx->scan_sms : ctx->sm_count, st));
    if (j->d_forced) CK(launch_append_keys(j->d_forced, j->forced_keys.size(), j->d_cand, j->cand_cap, &j->d_counters[CTR_CANDIDATES], st));
    CK(cudaEventRecord(j->ev[EV_SCAN], st));
    // candidates -> sorted by (stream, position)
    size_t tb = j->temp_bytes;
    CK(cub::DeviceRadixSort::SortKeys(j->d_temp, tb, j->d_cand, j->d_cand_sorted, (int)j->cand_cap, 0, 64, st));
    if (j->profiling) CK(cudaEventRecord(j->ev[EV_SORT], st));
    // K2
    ResolveArgs ra;
    ra.keys_sorted = j->d_cand_sorted; ra.cand_count = &j->d_counters[CTR_CANDIDATES]; ra.cand_cap = j->cand_cap; ra.len = j->d_len;
    ra.n_streams = n; ra.cmin = j->cfg.min; ra.cmax = j->cfg.max; ra.eof = j->eof; ra.counts = j->d_counts;
    ra.chunk_first = j->d_chunk_first; ra.chunks = j->d_chunks; ra.chunk_cap = j->chunk_cap; ra.consumed = j->d_consumed;
    ra.n_chunks = &j->d_counters[CTR_CHUNKS];
    CK(launch_resolve(ra, st));
    CK(cudaEventRecord(j->ev[EV_RESOLVE], st));
    return PBSGPU_OK;
}

// back half: K3 SHA-256 (hybrid launch) -> K4 probe + insert (when a set is attached) -> pack -> D2H of the results
int pbsgpu_job_enqueue_back(pbsgpu_job *j) {
    pbsgpu_ctx *ctx = j->ctx;
    cudaStream_t st = j->st;
    const uint32_t n = j->n;
    size_t tb = j->temp_bytes;
    bool early = false;
    if (j->ss != st) CK(cudaStreamWaitEvent(st, j->ev[EV_RESOLVE], 0));   // the chunk list comes from the scan partition
    if (j->profiling) CK(cudaEventRecord(j->ev[EV_BACK], st));
    if (j->want_digests && j->chunk_cap) {
        CK(launch_len_keys(j->d_chunks, &j->d_counters[CTR_CHUNKS], j->chunk_cap, j->d_keys, j->d_vals, st));
        tb = j->temp_bytes;
        CK(cub::DeviceRadixSort::SortPairsDescending(j->d_temp, tb, j->d_keys, j->d_keys2, j->d_vals, j->d_vals2,
                                                     (int)j->chunk_cap, 0, 32, st));
        ShaArgs ha;
        ha.base = j->base; ha.off = j->d_off; ha.chunks = j->d_chunks; ha.order = j->d_vals2;
        ha.n_chunks = &j->d_counters[CTR_CHUNKS]; ha.chunk_cap = j->chunk_cap; ha.digests = j->d_digests;
        ha.n_head = nullptr; ha.part = 0;
        if (j->variant == 1) CK(launch_sha_simple(ha, st, j->sha_suffix));
        else if (!hybrid_for(ctx)) CK(launch_sha_tuned(ha, st, j->sha_suffix));
        else {
            // hybrid: chunks longer than 2.5 x avg (their serial chains bound the batch's makespan) run on
            // the latency-optimised split kernel on a forked stream, concurrently with the rest
            uint64_t thr64 = (uint64_t)j->cfg.avg * (uint64_t)ctx->tune.thr_x10 / 10;
            uint32_t thr = thr64 > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)thr64;
            // at most one latency CTA (32 chunks) per SM of the partition and job; the longest chunks first
            const unsigned long long max_head = (unsigned long long)ctx->tune.head_per_sm * (unsigned long long)(ctx->part_sms > 0 ? ctx->part_sms : 24);
            CK(launch_split_point(j->d_keys2, &j->d_counters[CTR_CHUNKS], j->chunk_cap, thr, max_head, &j->d_counters[CTR_HEAD], st));
            ha.n_head = &j->d_counters[CTR_HEAD];
            // early input release: the head chunks are copied to the arena and hashed from there
            // (the copy runs HERE, on the job's own stream and the big partition -- a few ms -- not on the side stream,
            // where it would queue behind the 0.3 s latency kernel of the slot's previous job)
            // (a fixed-cut job has no head chunks: its bulk pass is the whole job, so it takes no arena)
            early = j->early && !j->fixed_log2 && arena_reserve(j, st);
            if (early) {
                CK(launch_arena_plan(ha, &j->d_counters[CTR_HEAD], j->arena_len, j->d_arena_off, st));
                CK(launch_arena_gather(ha, ctx->arena + j->arena_lo, j->d_arena_off, ctx->sm_count, st));
                ha.arena = ctx->arena + j->arena_lo; ha.arena_off = j->d_arena_off;
            }
            CK(cudaEventRecord(j->ev[EV_FORK], st));
            CK(cudaStreamWaitEvent(j->st2, j->ev[EV_FORK], 0));
            ha.part = 1; CK(launch_sha_split(ha, ctx->tune.spread_kb, j->st2, j->sha_suffix));
            ha.arena = nullptr; ha.arena_off = nullptr;
            CK(cudaEventRecord(j->ev[EV_JOIN], j->st2));
            if (early) CK(cudaEventRecord(ctx->arena_recs.back().ev, j->st2));   // the region may be reused after this
            ha.part = 2; CK(launch_sha_tuned(ha, st, j->sha_suffix));
            CK(cudaEventRecord(j->ev[EV_BULK], st));
            if (early) {
                // the caller's buffer is free once the bulk pass and the gather are done -- provided the candidate buffer
                // did not overflow (then the job is rerun from the input; pbsgpu_batch_wait_input checks the count)
                CK(cudaMemcpyAsync(j->h_early, &j->d_counters[CTR_CANDIDATES], sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
                CK(cudaEventRecord(j->ev[EV_INPUT], st));
            } else CK(cudaStreamWaitEvent(st, j->ev[EV_JOIN], 0));
        }
    }
    j->early_active = early;
    // The job's tail -- K4 (fused probe + insert), pack, D2H -- runs on the context's ONE tail stream when a set is
    // attached: jobs that share a set are thereby ordered in submission order without holding each other's streams
    // (a job's own stream is free for the slot's next job as soon as its SHA-256 is done).  An early-release job always
    // takes the tail stream: its own stream must not wait ~0.3 s for the long chunks' chains.
    cudaStream_t ts = ((j->set && j->want_digests) || early) ? ctx->tail_stream : st;
    if (early) {
        CK(cudaStreamWaitEvent(ts, j->ev[EV_INPUT], 0));
        CK(cudaStreamWaitEvent(ts, j->ev[EV_JOIN], 0));
        CK(cudaEventRecord(j->ev[EV_SHA], ts));
    } else {
        CK(cudaEventRecord(j->ev[EV_SHA], st));
        if (ts != st) CK(cudaStreamWaitEvent(ts, j->ev[EV_SHA], 0));
    }
    if (j->set && j->want_digests) {
        int rc = pbsgpu_set_enqueue(j->set, j->d_digests, &j->d_counters[CTR_CHUNKS], j->chunk_cap, 1, &j->d_counters[CTR_CANDIDATES],
                                    j->cand_cap, j->d_hit, &j->d_counters[CTR_NEW], j->d_set_scratch, ts);
        if (rc) return rc;
    }
    if (j->profiling) CK(cudaEventRecord(j->ev[EV_SET], ts));
    if (j->want_digests)
        CK(launch_pack_chunks(j->d_chunks, j->d_digests, j->set ? j->d_hit : nullptr, &j->d_counters[CTR_CHUNKS], j->chunk_cap, j->d_out, ts));
    CK(cudaMemcpyAsync(j->h_counters, j->d_counters, CTR_HOST * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ts));
    if (j->want_digests)
        CK(cudaMemcpyAsync(j->h_out, j->d_out, sizeof(pbsgpu_chunk) * j->chunk_cap, cudaMemcpyDeviceToHost, ts));
    if (!j->eof && n) CK(cudaMemcpyAsync(j->h_consumed, j->d_consumed, n * 8, cudaMemcpyDeviceToHost, ts));
    CK(cudaEventRecord(j->ev[EV_END], ts));
    j->state = JOB_ENQUEUED;
    return PBSGPU_OK;
}

int pbsgpu_job_enqueue(pbsgpu_job *j) {
    int rc = pbsgpu_job_enqueue_front(j);
    if (rc) return rc;
    return pbsgpu_job_enqueue_back(j);
}

// dense candidates (adversarial / highly structured data): replace the candidate buffers by exactly sized ones
int pbsgpu_job_prepare_rerun(pbsgpu_job *j, unsigned long long nc) {
    pbsgpu_ctx *ctx = j->ctx;
    // K4 skipped itself on the device (its guard is this very counter), so the set is untouched: settle the bookkeeping
    // of the skipped pass
    job_settle_set(j);
    j->state = JOB_CREATED;
    ctx->dev.put(j->d_cand); ctx->dev.put(j->d_cand_sorted); ctx->dev.put(j->d_temp);
    j->d_cand = j->d_cand_sorted = nullptr; j->d_temp = nullptr;
    j->cand_cap = nc + nc / 8 + 4096;
    if (j->cand_cap >= (1ull << 31)) return fail(ctx, PBSGPU_ENOMEM, "candidate density too high (%llu candidates)", nc);
    j->d_cand = (uint64_t *)ctx->dev.get(j->cand_cap * 8);
    j->d_cand_sorted = (uint64_t *)ctx->dev.get(j->cand_cap * 8);
    j->temp_bytes = sort_temp_bytes(j);
    j->d_temp = ctx->dev.get(j->temp_bytes);
    if (!j->d_cand || !j->d_cand_sorted || !j->d_temp) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed (rerun)");
    j->reruns++;
    return PBSGPU_OK;
}

// Blocks until the job is done; reruns it with a larger candidate buffer if the
// (statistically sized) one overflowed -- results are exact either way.
int pbsgpu_job_finish(pbsgpu_job *j) {
    pbsgpu_ctx *ctx = j->ctx;
    if (j->state == JOB_FINISHED) return PBSGPU_OK;
    for (;;) {
        CK(cudaEventSynchronize(j->ev[EV_END]));
        const unsigned long long nc = j->h_counters[CTR_CANDIDATES];
        if (!pbsgpu_job_overflowed(j, nc)) break;
        int rc = pbsgpu_job_prepare_rerun(j, nc);
        if (rc == PBSGPU_OK) rc = pbsgpu_job_enqueue(j);
        if (rc) return rc;
    }
    job_settle_set(j);
    j->state = JOB_FINISHED;
    pbsgpu_timing &t = j->timing;
    t.bytes = j->total_bytes; t.chunks = j->h_counters[CTR_CHUNKS]; t.candidates = j->h_counters[CTR_CANDIDATES]; t.reruns = j->reruns;
    t.scan_launches = j->fixed_log2 ? 0 : 1;
    const bool hyb = j->variant == 0 && hybrid_for(ctx);
    t.sha_launches = j->want_digests ? (hyb ? 2 : 1) : 0;
    t.other_launches = 3 + (j->d_forced ? 1 : 0) + (j->want_digests ? 2 + (hyb ? 1 : 0) : 0) + (j->set ? 3 : 0) + (j->early_active ? 2 : 0);
    if (j->profiling) {
        cudaEventElapsedTime(&t.scan_ms, j->ev[EV_START], j->ev[EV_SCAN]);
        cudaEventElapsedTime(&t.sort_ms, j->ev[EV_SCAN], j->ev[EV_SORT]);
        cudaEventElapsedTime(&t.resolve_ms, j->ev[EV_SORT], j->ev[EV_RESOLVE]);
        cudaEventElapsedTime(&t.sha_ms, j->ev[EV_BACK], j->ev[EV_SHA]);
        cudaEventElapsedTime(&t.set_ms, j->ev[EV_SHA], j->ev[EV_SET]);
        cudaEventElapsedTime(&t.total_ms, j->ev[EV_START], j->ev[EV_END]);
        cudaEventElapsedTime(&t.scan_t0, ctx->epoch, j->ev[EV_START]);
        cudaEventElapsedTime(&t.scan_t1, ctx->epoch, j->ev[EV_SCAN]);
        cudaEventElapsedTime(&t.sha_t0, ctx->epoch, j->ev[EV_BACK]);
        cudaEventElapsedTime(&t.sha_t1, ctx->epoch, j->ev[EV_SHA]);
        if (j->want_digests && hyb && j->chunk_cap) {
            cudaEventElapsedTime(&t.sha_long_ms, j->ev[EV_FORK], j->ev[EV_JOIN]);
            cudaEventElapsedTime(&t.sha_bulk_ms, j->ev[EV_FORK], j->ev[EV_BULK]);
            (void)cudaGetLastError();
        }
    }
    return PBSGPU_OK;
}

static const pbsgpu_batch_opts NO_OPTS = {sizeof(pbsgpu_batch_opts), 0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, 0};
// The caller's options in the current layout.  A caller built against an older header passes that layout's size (the
// offset of `crypt`: plain digests; the offset of `fixed_size`: the chunker) and gets the fields it knows.
static int opts_read(pbsgpu_ctx *ctx, const pbsgpu_batch_opts *o, pbsgpu_batch_opts *out) {
    *out = NO_OPTS;
    if (!o) return PBSGPU_OK;
    if (o->size != sizeof(pbsgpu_batch_opts) && o->size != offsetof(pbsgpu_batch_opts, fixed_size) &&
        o->size != offsetof(pbsgpu_batch_opts, crypt))
        return fail(ctx, PBSGPU_EINVAL, "pbsgpu_batch_opts.size = %u, expected %zu", o->size, sizeof(pbsgpu_batch_opts));
    memcpy(out, o, o->size);
    if (out->flags & ~(uint32_t)PBSGPU_BATCH_EARLY_INPUT) return fail(ctx, PBSGPU_EINVAL, "pbsgpu_batch_opts.flags = 0x%x: unknown bits", out->flags);
    if (out->crypt && out->crypt->ctx != ctx) return fail(ctx, PBSGPU_EINVAL, "crypt belongs to another context");
    const uint32_t fs = out->fixed_size;
    if (fs && (fs < 4096u || fs > (16u << 20) || (fs & (fs - 1))))
        return fail(ctx, PBSGPU_EINVAL, "pbsgpu_batch_opts.fixed_size = %u: a power of two from 4 KiB to 16 MiB", fs);
    if (fs && out->n_forced) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries do not apply to fixed-size chunks");
    return PBSGPU_OK;
}

extern "C" int pbsgpu_batch_submit_ex(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base_dev, const uint64_t *off,
                                      const uint64_t *len, uint32_t n, const pbsgpu_batch_opts *opts, pbsgpu_job **job) {
    if (!ctx || !job || (n && (!off || !len))) return PBSGPU_EINVAL;
    Guard g(ctx);
    *job = nullptr;
    pbsgpu_batch_opts o;
    int rc = opts_read(ctx, opts, &o);
    if (rc) return rc;
    if (o.stream_xxh3) return fail(ctx, PBSGPU_EINVAL, "stream_xxh3 is a synchronous-form option");
    if (n && !pbsgpu_is_device_ptr(base_dev)) return fail(ctx, PBSGPU_EINVAL, "pbsgpu_batch_submit needs a device pointer");
    pbsgpu_job *j = nullptr;
    rc = pbsgpu_job_create(ctx, cfg, base_dev, off, len, n, 1, 1, o.set, o.forced_stream, o.forced_off, o.n_forced, &j, o.fixed_size);
    if (rc) return rc;
    j->early = (o.flags & PBSGPU_BATCH_EARLY_INPUT) != 0;
    j->sha_suffix = pbsgpu_crypt_id_key(o.crypt);
    rc = pbsgpu_job_enqueue(j);
    if (rc) { pbsgpu_job_release(j); return rc; }
    *job = j;
    return PBSGPU_OK;
}
extern "C" int pbsgpu_batch_submit(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base_dev, const uint64_t *off,
                                   const uint64_t *len, uint32_t n, pbsgpu_job **job) {
    return pbsgpu_batch_submit_ex(ctx, cfg, base_dev, off, len, n, nullptr, job);
}

extern "C" int pbsgpu_batch_wait(pbsgpu_job *j, pbsgpu_chunk *out, uint64_t cap, uint64_t *n_out, pbsgpu_timing *timing) {
    if (!j) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = j->ctx;
    Guard g(ctx);
    int rc = pbsgpu_job_finish(j);
    if (rc == PBSGPU_OK) {
        uint64_t nch = j->h_counters[CTR_CHUNKS];
        if (n_out) *n_out = nch;
        if (timing) *timing = j->timing;
        if (nch > cap || (nch && !out))   // the job stays valid: call again with room for *n_out records (or pbsgpu_batch_free)
            return fail(ctx, PBSGPU_ERANGE, "output capacity %llu < %llu chunks", (unsigned long long)cap, (unsigned long long)nch);
        if (nch) memcpy(out, j->h_out, nch * sizeof(pbsgpu_chunk));
    }
    pbsgpu_job_release(j);
    return rc;
}

// Early input release (PBSGPU_BATCH_EARLY_INPUT): 1 = the device no longer reads the caller's buffer, 0 = not yet.
// A job whose candidate buffer overflowed is rerun FROM THE INPUT: it reports 0 until pbsgpu_batch_wait_input or
// pbsgpu_batch_wait ran that rerun.
extern "C" int pbsgpu_batch_input_done(pbsgpu_job *j) {
    if (!j) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = j->ctx;
    Guard g(ctx);
    cudaError_t e = cudaEventQuery(j->ev[j->early_active ? EV_INPUT : EV_END]);
    if (e == cudaErrorNotReady) { (void)cudaGetLastError(); return 0; }
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, PBSGPU_ECUDA, "cudaEventQuery -> %s", cudaGetErrorString(e)); }
    const unsigned long long nc = j->early_active ? *j->h_early : j->h_counters[CTR_CANDIDATES];
    return pbsgpu_job_overflowed(j, nc) ? 0 : 1;
}
extern "C" int pbsgpu_batch_wait_input(pbsgpu_job *j) {
    if (!j) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = j->ctx;
    Guard g(ctx);
    if (j->early_active) {
        CK(cudaEventSynchronize(j->ev[EV_INPUT]));
        if (!pbsgpu_job_overflowed(j, *j->h_early)) return PBSGPU_OK;
    }
    return pbsgpu_job_finish(j);   // no early release (or a rerun is due): the input is free when the job is done
}

extern "C" void pbsgpu_batch_free(pbsgpu_job *j) {
    if (!j) return;
    Guard g(j->ctx);
    pbsgpu_job_sync(j);
    pbsgpu_job_release(j);
}

// ---------------------------------------------------------------------------
// Synchronous batch; host input is staged through device buffers, group by group,
// H2D of group k+1 overlapping the kernels of group k.
// ---------------------------------------------------------------------------
struct Group { uint32_t first, count; uint64_t bytes; uint64_t f_lo, f_hi; };

// Finishes and releases one job of the synchronous batch (j becomes NULL).  `first` is the job's first stream in the
// caller's numbering: its records go to out[*produced...] with `stream` rebased by it, and the XXH3 run `xr` (when
// stream_xxh3 is set) to stream_xxh3 + first.  *produced counts every record; those that do not fit into `cap` are not
// copied (the caller reports ERANGE).
static int batch_collect(pbsgpu_job *&j, uint32_t first, XxhRun *xr, uint64_t *stream_xxh3, pbsgpu_chunk *out, uint64_t cap,
                         uint64_t *produced) {
    int rc = pbsgpu_job_finish(j);
    if (stream_xxh3) { int rx = pbsgpu_xxh3_collect(j->ctx, xr, stream_xxh3 + first, j->st); if (rc == PBSGPU_OK) rc = rx; }
    if (rc == PBSGPU_OK) {
        const uint64_t nch = j->h_counters[CTR_CHUNKS];
        if (*produced + nch <= cap && nch) {
            memcpy(out + *produced, j->h_out, nch * sizeof(pbsgpu_chunk));
            if (first) for (uint64_t k = 0; k < nch; k++) out[*produced + k].stream += first;
        }
        *produced += nch;
    }
    pbsgpu_job_release(j);
    j = nullptr;
    return rc;
}

static int batch_host(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const uint8_t *base, const uint64_t *off,
                      const uint64_t *len, uint32_t n, const pbsgpu_batch_opts &o, pbsgpu_chunk *out, uint64_t cap, uint64_t *n_out) {
    size_t fr = 0, tot = 0;
    CK(cudaMemGetInfo(&fr, &tot));
    uint64_t stage = ctx->stage_bytes ? ctx->stage_bytes : std::min<uint64_t>(4ull << 30, fr / 16);
    auto al = [](uint64_t x) { return (x + 255) & ~255ull; };
    std::vector<Group> groups;
    {
        Group g{0, 0, 0, 0, 0};
        for (uint32_t i = 0; i < n; i++) {
            uint64_t b = al(len[i]);
            if (g.count && g.bytes + b > stage) { groups.push_back(g); g = Group{i, 0, 0, 0, 0}; }
            g.count++; g.bytes += b;
        }
        if (g.count) groups.push_back(g);
    }
    {   // suggested boundaries are sorted by stream: give every group its slice
        uint64_t k = 0;
        for (auto &g : groups) {
            g.f_lo = k;
            while (k < o.n_forced && o.forced_stream[k] < g.first + g.count) {
                if (o.forced_stream[k] < g.first) return fail(ctx, PBSGPU_EINVAL, "suggested boundaries not sorted by stream");
                k++;
            }
            g.f_hi = k;
        }
        if (k != o.n_forced) return fail(ctx, PBSGPU_EINVAL, "suggested boundary names stream %u of %u", o.forced_stream[k], n);
    }
    constexpr int NBUF = 6;   // staged groups in flight: their SHA tails overlap the next groups' copies
    uint64_t buf_bytes = 256;
    for (auto &g : groups) buf_bytes = std::max(buf_bytes, g.bytes);
    struct Bufs {   // returned to the pool on every exit path
        Pool &pool; uint8_t *p[NBUF] = {}; explicit Bufs(Pool &pl) : pool(pl) {}
        ~Bufs() { for (auto q : p) pool.put(q); }
    } bufs(ctx->dev);
    int nbuf = (int)std::min<size_t>(NBUF, groups.size());
    for (int b = 0; b < nbuf; b++) {
        bufs.p[b] = (uint8_t *)ctx->dev.get(buf_bytes);
        if (!bufs.p[b]) return fail(ctx, PBSGPU_ENOMEM, "staging buffer of %llu bytes failed", (unsigned long long)buf_bytes);
    }
    std::vector<pbsgpu_job *> jobs(groups.size(), nullptr);
    std::vector<XxhRun> xruns(groups.size());   // f2: per-file XXH3-64 from the same staged bytes
    std::vector<cudaEvent_t> copied(groups.size(), nullptr);
    for (auto &e : copied) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    int rc = PBSGPU_OK;
    uint64_t produced = 0;
    std::vector<uint32_t> fs;
    for (size_t gi = 0; gi < groups.size() && rc == PBSGPU_OK; gi++) {
        if (gi >= (size_t)nbuf) {   // frees the buffer we are about to reuse
            const size_t c = gi - nbuf;
            rc = batch_collect(jobs[c], groups[c].first, &xruns[c], o.stream_xxh3, out, cap, &produced);
            if (rc) break;
        }
        const Group &g = groups[gi];
        uint8_t *buf = bufs.p[gi % nbuf];
        std::vector<uint64_t> goff(g.count), glen(g.count);
        uint64_t pos = 0;
        for (uint32_t k = 0; k < g.count; k++) {
            uint32_t i = g.first + k;
            goff[k] = pos; glen[k] = len[i];
            if (len[i]) {
                cudaError_t e = cudaMemcpyAsync(buf + pos, base + off[i], len[i], cudaMemcpyHostToDevice, ctx->copy_stream);
                if (e != cudaSuccess) { (void)cudaGetLastError(); rc = fail(ctx, PBSGPU_ECUDA, "H2D copy failed: %s", cudaGetErrorString(e)); break; }
            }
            pos += al(len[i]);
        }
        if (rc) break;
        cudaEventRecord(copied[gi], ctx->copy_stream);
        fs.assign(o.forced_stream + g.f_lo, o.forced_stream + g.f_hi);
        for (auto &s : fs) s -= g.first;
        pbsgpu_job *j = nullptr;
        rc = pbsgpu_job_create(ctx, cfg, buf, goff.data(), glen.data(), g.count, 1, 1, o.set, fs.data(), o.forced_off + g.f_lo,
                               g.f_hi - g.f_lo, &j, o.fixed_size);
        if (rc) break;
        j->sha_suffix = pbsgpu_crypt_id_key(o.crypt);
        cudaStreamWaitEvent(j->ss, copied[gi], 0);
        rc = pbsgpu_job_enqueue(j);
        if (rc == PBSGPU_OK && o.stream_xxh3) rc = pbsgpu_xxh3_enqueue(ctx, buf, goff.data(), glen.data(), g.count, j->st, &xruns[gi]);
        if (rc) { pbsgpu_job_release(j); break; }
        jobs[gi] = j;
    }
    for (size_t gi = 0; gi < groups.size(); gi++)
        if (jobs[gi]) { int r = batch_collect(jobs[gi], groups[gi].first, &xruns[gi], o.stream_xxh3, out, cap, &produced); if (rc == PBSGPU_OK) rc = r; }
    cudaStreamSynchronize(ctx->copy_stream);
    for (auto &e : copied) if (e) cudaEventDestroy(e);
    if (n_out) *n_out = produced;
    return rc;
}

extern "C" int pbsgpu_chunk_digest_batch_ex(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                                            const uint64_t *len, uint32_t n, const pbsgpu_batch_opts *opts, pbsgpu_chunk *out,
                                            uint64_t cap, uint64_t *n_out) {
    if (!ctx || (n && (!off || !len || !base)) || (cap && !out)) return PBSGPU_EINVAL;
    Guard g(ctx);
    pbsgpu_batch_opts o;
    int rc = opts_read(ctx, opts, &o);
    if (rc) return rc;
    if (o.set && o.set->ctx != ctx) return fail(ctx, PBSGPU_EINVAL, "set belongs to another context");
    if (!o.fixed_size && !pbsgpu_cfg_ok(cfg)) return fail(ctx, PBSGPU_EINVAL, "invalid pbsgpu_cfg (use pbsgpu_config)");
    uint64_t produced = 0;
    if (n == 0) { if (n_out) *n_out = 0; return PBSGPU_OK; }
    if (pbsgpu_is_device_ptr(base)) {   // device input: one job over all streams
        pbsgpu_job *j = nullptr;
        rc = pbsgpu_job_create(ctx, cfg, base, off, len, n, 1, 1, o.set, o.forced_stream, o.forced_off, o.n_forced, &j, o.fixed_size);
        if (rc) return rc;
        j->sha_suffix = pbsgpu_crypt_id_key(o.crypt);
        XxhRun xr;
        rc = pbsgpu_job_enqueue(j);
        if (rc == PBSGPU_OK && o.stream_xxh3) rc = pbsgpu_xxh3_enqueue(ctx, (const uint8_t *)base, off, len, n, j->st, &xr);
        if (rc == PBSGPU_OK) rc = batch_collect(j, 0, &xr, o.stream_xxh3, out, cap, &produced);
        else pbsgpu_job_release(j);
    } else {
        rc = batch_host(ctx, cfg, (const uint8_t *)base, off, len, n, o, out, cap, &produced);
    }
    if (n_out) *n_out = produced;
    if (rc == PBSGPU_OK && produced > cap)
        rc = fail(ctx, PBSGPU_ERANGE, "output capacity %llu < %llu chunks", (unsigned long long)cap, (unsigned long long)produced);
    return rc;
}

extern "C" int pbsgpu_chunk_digest_batch_xxh3(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                                              const uint64_t *len, uint32_t n, pbsgpu_set *set, pbsgpu_chunk *out,
                                              uint64_t cap, uint64_t *n_out, uint64_t *stream_xxh3) {
    pbsgpu_batch_opts o = NO_OPTS;
    o.set = set; o.stream_xxh3 = stream_xxh3;
    return pbsgpu_chunk_digest_batch_ex(ctx, cfg, base, off, len, n, &o, out, cap, n_out);
}

extern "C" int pbsgpu_chunk_digest_batch(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                                         const uint64_t *len, uint32_t n, pbsgpu_set *set, pbsgpu_chunk *out,
                                         uint64_t cap, uint64_t *n_out) {
    return pbsgpu_chunk_digest_batch_xxh3(ctx, cfg, base, off, len, n, set, out, cap, n_out, nullptr);
}

extern "C" int pbsgpu_scan_batch(pbsgpu_ctx *ctx, const pbsgpu_cfg *cfg, const void *base, const uint64_t *off,
                                 const uint64_t *len, uint32_t n, uint64_t *ends, uint64_t cap, uint64_t *stream_first,
                                 uint64_t *n_out) {
    if (!ctx || (n && (!off || !len || !base)) || !stream_first) return PBSGPU_EINVAL;
    Guard g(ctx);
    if (!pbsgpu_is_device_ptr(base) && n) return fail(ctx, PBSGPU_EINVAL, "pbsgpu_scan_batch needs a device pointer");
    pbsgpu_job *j = nullptr;
    int rc = pbsgpu_job_create(ctx, cfg, base, off, len, n, 1, 0, nullptr, nullptr, nullptr, 0, &j);
    if (rc) return rc;
    rc = pbsgpu_job_enqueue(j);
    if (rc == PBSGPU_OK) rc = pbsgpu_job_finish(j);
    if (rc == PBSGPU_OK) {
        uint64_t nch = j->h_counters[CTR_CHUNKS];
        if (n_out) *n_out = nch;
        if (nch > cap) rc = fail(ctx, PBSGPU_ERANGE, "output capacity %llu < %llu chunks", (unsigned long long)cap, (unsigned long long)nch);
        else {
            std::vector<ChunkRef> refs(nch);
            std::vector<uint64_t> first(n + 1);
            cudaError_t e = cudaMemcpy(refs.data(), j->d_chunks, nch * sizeof(ChunkRef), cudaMemcpyDeviceToHost);
            if (e == cudaSuccess) e = cudaMemcpy(first.data(), j->d_chunk_first, (n + 1) * 8, cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) { (void)cudaGetLastError(); rc = fail(ctx, PBSGPU_ECUDA, "D2H: %s", cudaGetErrorString(e)); }
            else {
                for (uint64_t k = 0; k < nch; k++) ends[k] = refs[k].start + refs[k].len;
                memcpy(stream_first, first.data(), (n + 1) * 8);
            }
        }
    }
    pbsgpu_job_release(j);
    return rc;
}

// ---------------------------------------------------------------------------
extern "C" int pbsgpu_corpus_fill(pbsgpu_ctx *ctx, const pbsgpu_corpus *c, uint64_t first_file, uint32_t n_files,
                                  void *dst_dev, uint64_t stride) {
    if (!ctx || !c || !dst_dev) return PBSGPU_EINVAL;
    Guard g(ctx);
    if (c->block_len == 0 || c->block_len % 8 || c->run_blocks == 0 || ((uintptr_t)dst_dev & 7) || (stride & 7) ||
        stride < c->file_len)
        return fail(ctx, PBSGPU_EINVAL, "corpus: block_len %% 8, run_blocks >= 1, 8-byte aligned dst/stride >= file_len required");
    CK(launch_corpus_fill(*c, first_file, n_files, (uint8_t *)dst_dev, stride, ctx->streams[0]));
    CK(cudaStreamSynchronize(ctx->streams[0]));
    return PBSGPU_OK;
}
