// pbs_plus_b200/csrc/capi_set.cu -- C ABI of the known-digest set (K4) and its multi-GPU merge over NCCL.
//
// Replaces the known-chunk bookkeeping of the reference's dedup session (seeded from the previous snapshot:
// backupproxy.PreviousBackupRef, reference internal/pxarmount/commit.go:286-294, origPayloadIdx commit.go:324-329;
// "Only new chunks are uploaded", docs/pxar-mount.md:105).  The table lives on the device; operations are ordered by
// a completion event so that batch jobs on different CUDA streams can probe + insert as part of their own pipeline.
#include <dlfcn.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <cub/device/device_radix_sort.cuh>

#include "host.hpp"

using namespace pbsgpu;

static int set_alloc_table(pbsgpu_ctx *ctx, uint64_t cap, SetTable *t, cudaStream_t st) {
    t->cap = cap;
    t->tags = (uint64_t *)ctx->dev.get(cap * 8);
    t->keys = (uint64_t *)ctx->dev.get(cap * 32);
    if (!t->tags || !t->keys) {
        ctx->dev.put(t->tags); ctx->dev.put(t->keys); t->tags = t->keys = nullptr;
        return fail(ctx, PBSGPU_ENOMEM, "digest set allocation failed (%llu slots)", (unsigned long long)cap);
    }
    CK(cudaMemsetAsync(t->tags, 0, cap * 8, st));
    return PBSGPU_OK;
}

extern "C" int pbsgpu_set_create(pbsgpu_ctx *ctx, uint64_t capacity_hint, pbsgpu_set **out) {
    if (!ctx || !out) return PBSGPU_EINVAL;
    Guard g(ctx);
    uint64_t cap = 1024;
    while (cap < capacity_hint * 2) cap <<= 1;
    pbsgpu_set *s = new pbsgpu_set();
    s->ctx = ctx; s->count = 0; s->pending_max = 0;
    int rc = set_alloc_table(ctx, cap, &s->t, ctx->streams[0]);
    if (rc == PBSGPU_OK && cudaEventCreateWithFlags(&s->last, cudaEventDisableTiming) != cudaSuccess) rc = fail(ctx, PBSGPU_ECUDA, "cudaEventCreate failed");
    if (rc == PBSGPU_OK && cudaStreamSynchronize(ctx->streams[0]) != cudaSuccess) rc = fail(ctx, PBSGPU_ECUDA, "digest set initialisation failed");
    if (rc) { (void)cudaGetLastError(); ctx->dev.put(s->t.tags); ctx->dev.put(s->t.keys); if (s->last) cudaEventDestroy(s->last); delete s; return rc; }
    *out = s;
    return PBSGPU_OK;
}
extern "C" void pbsgpu_set_destroy(pbsgpu_set *s) {
    if (!s) return;
    Guard g(s->ctx);
    if (s->last_valid) cudaEventSynchronize(s->last);
    cudaStreamSynchronize(s->ctx->streams[0]);
    s->ctx->dev.put(s->t.tags); s->ctx->dev.put(s->t.keys);
    if (s->last) cudaEventDestroy(s->last);
    delete s;
}
// Digests in the table as far as finished operations go (a fused batch probe counts once its job was collected).
extern "C" int pbsgpu_set_count(pbsgpu_set *s, uint64_t *count) { if (!s || !count) return PBSGPU_EINVAL; *count = s->count; return 0; }

// Capacity rule.  Insertions never fail as long as the table has a free slot, so the HARD requirement is
//     count + pending_max + more <= 7/8 * cap        (pending_max = worst-case insertions of operations still in flight)
// and the COMFORT target is a load <= 50 % of what is really in the table (count).  The worst case of a fused batch
// probe is its launch bound (bytes / min chunk size), 3.6 x what random data produces -- using it for the comfort
// target made the table grow (and the host wait for every operation in flight) in the middle of a pipelined run.
// Rehashing waits for every operation enqueued on the table.
static int set_reserve(pbsgpu_set *s, uint64_t more, cudaStream_t st) {
    pbsgpu_ctx *ctx = s->ctx;
    const uint64_t hard = s->count + s->pending_max + more;
    const uint64_t soft = s->count + (s->pending_max + more) / 4;
    if (hard <= s->t.cap / 8 * 7 && soft * 2 <= s->t.cap) return PBSGPU_OK;
    uint64_t cap = s->t.cap;
    while (hard > cap / 8 * 7 || soft * 2 > cap) cap <<= 1;
    if (s->last_valid) CK(cudaEventSynchronize(s->last));
    SetTable nt;
    int rc = set_alloc_table(ctx, cap, &nt, st);
    if (rc) return rc;
    CK(launch_set_rehash(s->t, nt, st));
    CK(cudaStreamSynchronize(st));
    ctx->dev.put(s->t.tags); ctx->dev.put(s->t.keys);
    s->t = nt;
    return PBSGPU_OK;
}

// scratch layout of one operation: tag[cap] tag2[cap] (u64) | idx[cap] idx2[cap] (u32) | miss[cap] | cub temp
struct SetLayout { size_t tag, tag2, idx, idx2, miss, temp, temp_bytes, total; };
static SetLayout set_layout(uint64_t cap) {
    SetLayout L;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t tb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (int)std::max<uint64_t>(cap, 1));
    L.tag = 0; L.tag2 = al(L.tag + cap * 8); L.idx = al(L.tag2 + cap * 8); L.idx2 = al(L.idx + cap * 4);
    L.miss = al(L.idx2 + cap * 4); L.temp = al(L.miss + cap); L.temp_bytes = tb + 256; L.total = L.temp + L.temp_bytes;
    return L;
}
size_t pbsgpu_set_scratch_bytes(uint64_t cap) { return set_layout(cap).total; }

int pbsgpu_set_enqueue(pbsgpu_set *s, const uint8_t *d_dig, const unsigned long long *n_dev, uint64_t cap, int do_insert,
                       const unsigned long long *guard, uint64_t guard_max, uint8_t *d_hit, unsigned long long *d_new,
                       void *scratch, cudaStream_t st) {
    pbsgpu_ctx *ctx = s->ctx;
    if (cap == 0) return PBSGPU_OK;
    if (cap >= (1ull << 31)) return fail(ctx, PBSGPU_EINVAL, "too many digests in one call");
    if (do_insert) { int rc = set_reserve(s, cap, ctx->streams[0]); if (rc) return rc; }
    if (s->last_valid) CK(cudaStreamWaitEvent(st, s->last, 0));   // table operations are totally ordered
    const SetLayout L = set_layout(cap);
    uint8_t *b = (uint8_t *)scratch;
    uint64_t *tag = (uint64_t *)(b + L.tag), *tag2 = (uint64_t *)(b + L.tag2);
    uint32_t *idx = (uint32_t *)(b + L.idx), *idx2 = (uint32_t *)(b + L.idx2);
    size_t tb = L.temp_bytes;
    CK(launch_set_make_keys(d_dig, n_dev, cap, tag, idx, st));
    CK(cub::DeviceRadixSort::SortPairs(b + L.temp, tb, tag, tag2, idx, idx2, (int)cap, 0, 64, st));   // stable
    CK(launch_set_mark_probe_insert(s->t, d_dig, tag2, idx2, n_dev, cap, guard, guard_max, do_insert, d_hit, b + L.miss, d_new, st));
    CK(cudaEventRecord(s->last, st));
    s->last_valid = true;
    if (do_insert) s->pending_max += cap;
    return PBSGPU_OK;
}

void pbsgpu_set_reconcile(pbsgpu_set *s, uint64_t cap, uint64_t n_new) {
    s->pending_max = s->pending_max >= cap ? s->pending_max - cap : 0;
    s->count += n_new;
}

// d_dig: device pointer to n*32 bytes.  d_hit: device n bytes or NULL.  Synchronous (count known on return).
int pbsgpu_set_process_dev(pbsgpu_set *s, const uint8_t *d_dig, uint64_t n, int do_insert, uint8_t *d_hit) {
    pbsgpu_ctx *ctx = s->ctx;
    if (n == 0) return PBSGPU_OK;
    if (n >= (1ull << 31)) return fail(ctx, PBSGPU_EINVAL, "too many digests in one call");
    Blocking b(ctx, ctx->streams[0]);
    void *scratch = b.get<uint8_t>(pbsgpu_set_scratch_bytes(n));
    unsigned long long *d_new = b.get<unsigned long long>(1), h_new = 0;
    if (!scratch || !d_new) return fail(ctx, PBSGPU_ENOMEM, "digest set scratch allocation failed");
    b.e = cudaMemsetAsync(d_new, 0, 8, b.st);
    if (!b.ok()) return b.finish("digest set");
    if (int rc = pbsgpu_set_enqueue(s, d_dig, nullptr, n, do_insert, nullptr, 0, d_hit, d_new, scratch, b.st)) return rc;
    b.e = cudaMemcpyAsync(&h_new, d_new, 8, cudaMemcpyDeviceToHost, b.st);
    const int rc = b.finish("digest set");
    pbsgpu_set_reconcile(s, do_insert ? n : 0, rc ? 0 : h_new);   // the enqueue added n to pending_max
    return rc;
}

static int set_process(pbsgpu_set *s, const uint8_t *d32, uint64_t n, int do_insert, uint8_t *hit_host) {
    if (!s || (n && !d32)) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    if (n == 0) return PBSGPU_OK;
    Blocking b(ctx, ctx->streams[0]);
    const uint64_t zero = 0, bytes = n * 32;
    const uint8_t *d_dig;
    if (int rc = b.stage(d32, &zero, &bytes, 1, &d_dig)) return rc;
    uint8_t *d_hit = hit_host ? b.get<uint8_t>(n) : nullptr;
    if (hit_host && !d_hit) return fail(ctx, PBSGPU_ENOMEM, "hit flag allocation failed");
    int rc = pbsgpu_set_process_dev(s, d_dig, n, do_insert, d_hit);
    if (rc == PBSGPU_OK && hit_host) {
        b.e = cudaMemcpyAsync(hit_host, d_hit, n, cudaMemcpyDeviceToHost, b.st);
        rc = b.finish("hit copy");
    }
    return rc;
}
extern "C" int pbsgpu_set_insert(pbsgpu_set *s, const uint8_t *d32, uint64_t n, uint8_t *hit) { return set_process(s, d32, n, 1, hit); }
extern "C" int pbsgpu_set_probe(pbsgpu_set *s, const uint8_t *d32, uint64_t n, uint8_t *hit) { return set_process(s, d32, n, 0, hit); }

extern "C" int pbsgpu_set_seed_didx(pbsgpu_set *s, const uint8_t *didx, uint64_t size, uint64_t *n_entries) {
    if (!s || !didx) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    if (size < 4096 || (size - 4096) % 40) return fail(ctx, PBSGPU_EINVAL, "not a dynamic index image (size %llu)", (unsigned long long)size);
    uint64_t n = (size - 4096) / 40;
    std::vector<uint8_t> dig(n * 32);
    for (uint64_t i = 0; i < n; i++) memcpy(&dig[i * 32], didx + 4096 + i * 40 + 8, 32);
    if (n_entries) *n_entries = n;
    return set_process(s, dig.data(), n, 1, nullptr);
}

extern "C" int pbsgpu_set_seed_fidx(pbsgpu_set *s, const uint8_t *fidx, uint64_t bytes, uint64_t *n_entries) {
    if (!s || !fidx) return PBSGPU_EINVAL;
    uint64_t n = 0;
    if (int rc = pbsgpu_fidx_parse(s->ctx, fidx, bytes, nullptr, nullptr, nullptr, 0, &n, 0)) return rc;
    if (n_entries) *n_entries = n;
    return set_process(s, fidx + 4096, n, 1, nullptr);   // the digest table is contiguous: n x 32 bytes
}

// ---------------------------------------------------------------------------
// e: multi-GPU merge.  NCCL is resolved at run time (dlopen) so that libpbsgpu.so has no link-time dependency on it:
// single-GPU users never need libnccl, and a host that already loaded one (torch's bundled libnccl.so.2) shares it.
// ---------------------------------------------------------------------------
namespace {
typedef int ncclResult;
typedef struct { char internal[128]; } ncclUniqueId_t;
struct Nccl {
    void *h = nullptr;
    ncclResult (*GetUniqueId)(ncclUniqueId_t *) = nullptr;
    ncclResult (*CommInitRank)(void **, int, ncclUniqueId_t, int) = nullptr;
    ncclResult (*CommDestroy)(void *) = nullptr;
    ncclResult (*CommCount)(const void *, int *) = nullptr;
    ncclResult (*CommUserRank)(const void *, int *) = nullptr;
    ncclResult (*AllGather)(const void *, void *, size_t, int /*ncclDataType_t*/, void *, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult) = nullptr;
    std::string why;
};
Nccl *nccl() {
    static Nccl N;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *names[] = {getenv("PBSGPU_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char *nm : names) {
            if (!nm || !*nm) continue;
            N.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (N.h) break;
            N.why = dlerror() ? dlerror() : "dlopen failed";
        }
        if (!N.h) { if (N.why.empty()) N.why = "libnccl.so.2 not found (set PBSGPU_NCCL_LIB)"; return; }
        auto sym = [&](const char *s) { return dlsym(N.h, s); };
        N.GetUniqueId = (decltype(N.GetUniqueId))sym("ncclGetUniqueId");
        N.CommInitRank = (decltype(N.CommInitRank))sym("ncclCommInitRank");
        N.CommDestroy = (decltype(N.CommDestroy))sym("ncclCommDestroy");
        N.CommCount = (decltype(N.CommCount))sym("ncclCommCount");
        N.CommUserRank = (decltype(N.CommUserRank))sym("ncclCommUserRank");
        N.AllGather = (decltype(N.AllGather))sym("ncclAllGather");
        N.GetErrorString = (decltype(N.GetErrorString))sym("ncclGetErrorString");
        if (!N.GetUniqueId || !N.CommInitRank || !N.CommDestroy || !N.CommCount || !N.CommUserRank || !N.AllGather) {
            N.why = "libnccl lacks a required symbol"; dlclose(N.h); N.h = nullptr;
        }
    });
    return &N;
}
constexpr int NCCL_UINT8 = 1, NCCL_UINT64 = 5;   // ncclDataType_t values (stable across NCCL 2.x)
}  // namespace

extern "C" int pbsgpu_nccl_unique_id(uint8_t id[128]) {
    if (!id) return PBSGPU_EINVAL;
    Nccl *N = nccl();
    if (!N->h) return PBSGPU_ENODEV;
    ncclUniqueId_t u;
    if (N->GetUniqueId(&u) != 0) return PBSGPU_ECUDA;
    memcpy(id, u.internal, 128);
    return PBSGPU_OK;
}
extern "C" int pbsgpu_nccl_comm_create(pbsgpu_ctx *ctx, const uint8_t id[128], int nranks, int rank, void **comm) {
    if (!ctx || !id || !comm || nranks < 1 || rank < 0 || rank >= nranks) return PBSGPU_EINVAL;
    Guard g(ctx);
    Nccl *N = nccl();
    if (!N->h) return fail(ctx, PBSGPU_ENODEV, "NCCL unavailable: %s", N->why.c_str());
    ncclUniqueId_t u;
    memcpy(u.internal, id, 128);
    void *c = nullptr;
    ncclResult r = N->CommInitRank(&c, nranks, u, rank);
    if (r != 0) return fail(ctx, PBSGPU_ECUDA, "ncclCommInitRank: %s", N->GetErrorString ? N->GetErrorString(r) : "error");
    *comm = c;
    return PBSGPU_OK;
}
extern "C" void pbsgpu_nccl_comm_destroy(void *comm) {
    Nccl *N = nccl();
    if (comm && N->h) N->CommDestroy(comm);
}

extern "C" int pbsgpu_set_allgather(pbsgpu_set *s, void *comm, const uint8_t *d32, uint64_t n, uint8_t *hit) {
    if (!s || !comm || (n && !d32)) return PBSGPU_EINVAL;
    pbsgpu_ctx *ctx = s->ctx;
    Guard g(ctx);
    Nccl *N = nccl();
    if (!N->h) return fail(ctx, PBSGPU_ENODEV, "NCCL unavailable: %s", N->why.c_str());
    int world = 0, rank = 0;
    if (N->CommCount(comm, &world) != 0 || N->CommUserRank(comm, &rank) != 0 || world < 1) return fail(ctx, PBSGPU_EINVAL, "bad NCCL communicator");
    Blocking b(ctx, ctx->streams[0]);
    if (s->last_valid) CK(cudaStreamWaitEvent(b.st, s->last, 0));
    auto ncclck = [&](ncclResult r, const char *what) {
        return r == 0 ? PBSGPU_OK : fail(ctx, PBSGPU_ECUDA, "%s: %s", what, N->GetErrorString ? N->GetErrorString(r) : "NCCL error");
    };
    // 1. counts (one u64 per rank); the payload is padded to the largest, so the host needs them
    uint64_t *d_counts = b.get<uint64_t>(world);
    if (!d_counts) return fail(ctx, PBSGPU_ENOMEM, "allgather: allocation failed");
    std::vector<uint64_t> h_counts(world);
    b.e = cudaMemcpyAsync(d_counts + rank, &n, 8, cudaMemcpyHostToDevice, b.st);
    if (!b.ok()) return b.finish("allgather counts");
    int rc = ncclck(N->AllGather(d_counts + rank, d_counts, 1, NCCL_UINT64, comm, b.st), "ncclAllGather(counts)");
    if (rc) return rc;
    b.e = cudaMemcpyAsync(h_counts.data(), d_counts, (size_t)world * 8, cudaMemcpyDeviceToHost, b.st);
    rc = b.finish("allgather counts");
    if (rc) return rc;
    uint64_t max_n = 0, total = 0, first = 0;
    for (int r = 0; r < world; r++) { max_n = std::max(max_n, h_counts[r]); if (r < rank) first += h_counts[r]; total += h_counts[r]; }
    if (total == 0) return PBSGPU_OK;
    if (total >= (1ull << 31)) return fail(ctx, PBSGPU_EINVAL, "too many digests in one merge");
    // 2. payload, padded to max_n rows per rank, then compacted into global (rank, index) order
    uint8_t *padded = b.get<uint8_t>((uint64_t)world * max_n * 32), *dense = b.get<uint8_t>(total * 32), *d_hit = b.get<uint8_t>(total);
    if (!padded || !dense || !d_hit) return fail(ctx, PBSGPU_ENOMEM, "allgather: allocation of %llu digests failed", (unsigned long long)total);
    uint8_t *slot = padded + (size_t)rank * max_n * 32;
    if (n) b.e = cudaMemcpyAsync(slot, d32, n * 32, pbsgpu_is_device_ptr(d32) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, b.st);
    if (!b.ok()) return b.finish("allgather digests");
    rc = ncclck(N->AllGather(slot, padded, max_n * 32, NCCL_UINT8, comm, b.st), "ncclAllGather(digests)");
    if (rc) return rc;
    b.e = launch_set_compact_gather(padded, d_counts, (uint32_t)world, max_n, dense, b.st);
    if (!b.ok()) return b.finish("allgather compaction");
    // 3. every rank inserts everything in the same order: replicas stay identical, flags equal a single-GPU run
    rc = pbsgpu_set_process_dev(s, dense, total, 1, d_hit);
    if (rc == PBSGPU_OK && hit && n) {
        b.e = cudaMemcpyAsync(hit, d_hit + first, n, cudaMemcpyDeviceToHost, b.st);
        rc = b.finish("hit copy");
    }
    return rc;
}
