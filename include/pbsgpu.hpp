// pbsgpu.hpp -- C++ host mirror of the reference's Go surface for the hot path, over the C ABI.
//
// The reference is compiled Go and the build image has no Go toolchain, so the host side above
// the C ABI is written in C++ (header only).  Names, argument meaning and error behaviour follow
// the Go call sites in the reference (internal/pxarmount/commit.go):
//     buzhash.NewConfig(4096)                                   :302-305
//     transfer.NewRemoteDedupSplitArchiveWriter(..., origPayloadIdx)   :329
//     writer.WriteEntryReader(entry, reader, size)               :720, :858
//     writer.Finish()                                            :383
// Go `error` returns become pbsgpu::Error exceptions carrying the same text a Go caller would wrap.
#pragma once
#include <sys/random.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "pbsgpu.h"

namespace pbsgpu {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

namespace buzhash {
using Config = pbsgpu_cfg;
// buzhash.NewConfig(avgKiB) (Config, error)
inline Config NewConfig(int avg_kib) {
    Config c;
    int rc = pbsgpu_config_kib((uint32_t)avg_kib, nullptr, &c);
    if (rc) throw Error(rc, "buzhash: invalid average chunk size " + std::to_string(avg_kib) + " KiB");
    return c;
}
}  // namespace buzhash

class Engine {
  public:
    explicit Engine(int device = 0) {
        int rc = pbsgpu_open(device, &ctx_);
        if (rc) throw Error(rc, "pbsgpu_open: no usable CUDA device (there is no CPU fallback)");
    }
    ~Engine() { pbsgpu_close(ctx_); }
    Engine(const Engine &) = delete;
    Engine &operator=(const Engine &) = delete;
    pbsgpu_ctx *ctx() const { return ctx_; }
    void check(int rc) const { if (rc) throw Error(rc, std::string("pbsgpu: ") + pbsgpu_strerror(ctx_)); }

  private:
    pbsgpu_ctx *ctx_ = nullptr;
};

class KnownSet {   // the session's known-chunk set (PreviousBackupRef, commit.go:286-294)
  public:
    explicit KnownSet(Engine &e, uint64_t hint = 1 << 16) : e_(e) { e.check(pbsgpu_set_create(e.ctx(), hint, &s_)); }
    ~KnownSet() { pbsgpu_set_destroy(s_); }
    pbsgpu_set *handle() const { return s_; }
    uint64_t SeedFromDidx(const std::vector<uint8_t> &didx) {   // origPayloadIdx, commit.go:324-328
        uint64_t n = 0;
        if (!didx.empty()) e_.check(pbsgpu_set_seed_didx(s_, didx.data(), didx.size(), &n));
        return n;
    }
    uint64_t SeedFromFidx(const std::vector<uint8_t> &fidx) {   // the previous snapshot's index of the same disk image
        uint64_t n = 0;
        e_.check(pbsgpu_set_seed_fidx(s_, fidx.data(), fidx.size(), &n));
        return n;
    }
    uint64_t size() const { uint64_t c = 0; pbsgpu_set_count(s_, &c); return c; }

  private:
    Engine &e_;
    pbsgpu_set *s_ = nullptr;
};

// Encrypt mode (BackupConfig's CryptMode, commit.go:314): one 32-byte client key on the engine's device.  The writers
// below take it to produce keyed digests and, for the payload stream, encrypted blobs.
class CryptConfig {
  public:
    CryptConfig(Engine &e, const uint8_t key[32]) { e.check(pbsgpu_crypt_create(e.ctx(), key, &c_)); }
    ~CryptConfig() { pbsgpu_crypt_destroy(c_); }   // zeroes the key material
    CryptConfig(const CryptConfig &) = delete;
    CryptConfig &operator=(const CryptConfig &) = delete;
    const pbsgpu_crypt *handle() const { return c_; }

  private:
    pbsgpu_crypt *c_ = nullptr;
};

namespace transfer {

struct Entry { std::string Path; uint64_t FileSize; };   // the fields of pxar.Entry the hot path reads
struct IndexRecord { std::string path; uint64_t end_off; uint8_t digest[32]; bool known; };
// io.Reader: fill buf[0..n) and return the number of bytes produced (0 = EOF)
using Reader = std::function<size_t(uint8_t *buf, size_t n)>;

class DedupWriter {
  public:
    // crypt (may be NULL): the index holds keyed digests
    DedupWriter(Engine &e, const buzhash::Config &cfg, KnownSet *known, uint64_t staging_bytes = 1ull << 30,
                const CryptConfig *crypt = nullptr)
        : e_(e), cfg_(cfg), known_(known), crypt_(crypt), cap_(staging_bytes) {
        buf_ = (uint8_t *)pbsgpu_host_alloc(e.ctx(), cap_);
        if (!buf_) throw Error(PBSGPU_ENOMEM, "pbsgpu: pinned staging allocation failed");
    }
    ~DedupWriter() { pbsgpu_host_free(e_.ctx(), buf_); }

    // writer.WriteEntryReader(entry, reader, size): pulls exactly `size` bytes (io.ReadFull semantics)
    void WriteEntryReader(const Entry &entry, const Reader &reader, uint64_t size) {
        if (finished_) throw Error(PBSGPU_ESTATE, "transfer: writer already finished");
        uint64_t start = (fill_ + 255) & ~255ull;
        if (start + size > cap_) { Flush(); start = 0; }
        if (size > cap_) throw Error(PBSGPU_ENOMEM, "transfer: entry larger than the staging buffer: " + entry.Path);
        uint64_t got = 0;
        while (got < size) {
            size_t k = reader(buf_ + start + got, size - got);
            if (k == 0) throw Error(PBSGPU_EINVAL, "transfer: short read for " + entry.Path + ": unexpected EOF");
            got += k;
        }
        entries_.push_back(entry); off_.push_back(start); len_.push_back(size);
        fill_ = start + size;
    }
    void Flush() {
        if (entries_.empty()) return;
        uint64_t cap = entries_.size();
        for (uint64_t l : len_) cap += l / (cfg_.min > 64 ? cfg_.min : 65);
        std::vector<pbsgpu_chunk> out(cap + 1);
        std::vector<uint64_t> xxh(entries_.size());
        uint64_t n = 0;
        pbsgpu_batch_opts o = {sizeof(pbsgpu_batch_opts), 0, known_ ? known_->handle() : nullptr, nullptr, nullptr, 0,
                               xxh.data(), crypt_ ? crypt_->handle() : nullptr, 0};
        e_.check(pbsgpu_chunk_digest_batch_ex(e_.ctx(), &cfg_, buf_, off_.data(), len_.data(), (uint32_t)entries_.size(), &o,
                                              out.data(), out.size(), &n));
        for (size_t i = 0; i < entries_.size(); i++) backed_hashes_[entries_[i].Path] = xxh[i];
        for (uint64_t i = 0; i < n; i++) {
            IndexRecord r;
            r.path = entries_[out[i].stream].Path; r.end_off = out[i].end_off;
            std::memcpy(r.digest, out[i].digest, 32); r.known = (out[i].flags & PBSGPU_CHUNK_KNOWN) != 0;
            index_.push_back(r);
        }
        entries_.clear(); off_.clear(); len_.clear(); fill_ = 0;
    }
    const std::vector<IndexRecord> &Finish() { Flush(); finished_ = true; return index_; }
    // relPath -> XXH3-64 of the uploaded bytes: commitWalkState.backedHashes (commit.go:187, :725)
    const std::map<std::string, uint64_t> &BackedHashes() const { return backed_hashes_; }

  private:
    Engine &e_;
    buzhash::Config cfg_;
    KnownSet *known_;
    const CryptConfig *crypt_;
    uint8_t *buf_ = nullptr;
    uint64_t cap_, fill_ = 0;
    bool finished_ = false;
    std::vector<Entry> entries_;
    std::vector<uint64_t> off_, len_;
    std::vector<IndexRecord> index_;
    std::map<std::string, uint64_t> backed_hashes_;
};

// ---- the layout-faithful writer: ONE pxar v2 payload stream through pbsgpu_stream_* ---------------------------------
// Start marker, then per file a 16-byte PAYLOAD header + content (reference internal/pxarmount/pxarfs.go:408-411),
// chunker state carried across files, a suggested boundary at every file start, bytes read straight into the
// library's pinned ring.  WriteEntryReader (commit.go:720) returns the entry's payload offset.
// Optional: `blob_mode` (PBSGPU_BLOB_RAW .. _LZH, _LZL, _LZC) hands the DataBlob of every new chunk to `upload_blob(digest, blob,
// len)`, encoded on the GPU from the stream's windows; `hash_files` records every file's XXH3-64 in BackedHashes()
// (commitWalkState.backedHashes, commit.go:725); `crypt` gives keyed digests and encrypted blobs, their IVs drawn from the
// OS CSPRNG by the stream.
struct PayloadChunk { uint64_t end_off; uint8_t digest[32]; bool known; };
using UploadBlob = std::function<void(const uint8_t digest[32], const uint8_t *blob, uint64_t len)>;

class PayloadStreamWriter {
  public:
    PayloadStreamWriter(Engine &e, const buzhash::Config &cfg, KnownSet *known, bool suggest = true,
                        int blob_mode = PBSGPU_BLOB_NONE, UploadBlob upload_blob = nullptr, bool hash_files = false,
                        const CryptConfig *crypt = nullptr)
        : e_(e), suggest_(suggest), upload_(std::move(upload_blob)), hash_(hash_files) {
        if ((blob_mode != PBSGPU_BLOB_NONE) != (upload_ != nullptr))
            throw Error(PBSGPU_EINVAL, "transfer: a blob mode and an upload_blob callback go together");
        if (upload_) blob_buf_.resize(pbsgpu_blob_size_enc(cfg.max) + (16u << 20));
        e.check(pbsgpu_stream_open(e.ctx(), &cfg, known ? known->handle() : nullptr, &s_));
        try {   // the destructor does not run for a constructor that throws
            if (crypt) e.check(pbsgpu_stream_crypt(s_, crypt->handle(), nullptr));
            if (upload_) e.check(pbsgpu_stream_blob_mode(s_, blob_mode));
            raw(header(0x834c68c2194a4ed2ull, 16));                 // PXAR_PAYLOAD_START_MARKER
        } catch (...) {
            pbsgpu_stream_close(s_);
            throw;
        }
    }
    ~PayloadStreamWriter() { pbsgpu_stream_close(s_); }
    PayloadStreamWriter(const PayloadStreamWriter &) = delete;
    PayloadStreamWriter &operator=(const PayloadStreamWriter &) = delete;

    uint64_t WriteEntryReader(const Entry &entry, const Reader &reader, uint64_t size) {
        if (finished_) throw Error(PBSGPU_ESTATE, "transfer: writer already finished");
        const uint64_t off = pbsgpu_stream_position(s_);
        if (suggest_) e_.check(pbsgpu_stream_suggest(s_, off));
        if (hash_) { e_.check(pbsgpu_stream_hash_range(s_, off + 16, size)); hashed_.push_back(entry.Path); }
        raw(header(0x28147a1b0b7c1a25ull, 16 + size));              // PXAR_PAYLOAD
        const uint64_t slot = pbsgpu_stream_slot_bytes(s_);
        uint64_t left = size;
        while (left) {
            void *p = nullptr;
            e_.check(pbsgpu_stream_reserve(s_, &p));
            const uint64_t want = left < slot ? left : slot;
            uint64_t got = 0;
            while (got < want) {
                size_t k = reader((uint8_t *)p + got, want - got);
                if (k == 0) { pbsgpu_stream_commit(s_, 0); throw Error(PBSGPU_EINVAL, "transfer: short read for " + entry.Path + ": unexpected EOF"); }
                got += k;
            }
            e_.check(pbsgpu_stream_commit(s_, want));
            left -= want;
        }
        drain();
        return off;
    }
    const std::vector<PayloadChunk> &Finish() {
        if (!finished_) {
            raw(header(0x6c72b78b984c81b5ull, 16));                 // PXAR_PAYLOAD_TAIL_MARKER
            e_.check(pbsgpu_stream_finish(s_));
            drain();
            finished_ = true;
        }
        return index_;
    }
    const std::map<std::string, uint64_t> &BackedHashes() const { return backed_hashes_; }

  private:
    static std::vector<uint8_t> header(uint64_t htype, uint64_t full) {
        std::vector<uint8_t> h(16);
        for (int i = 0; i < 8; i++) { h[i] = (uint8_t)(htype >> (8 * i)); h[8 + i] = (uint8_t)(full >> (8 * i)); }
        return h;
    }
    void raw(const std::vector<uint8_t> &b) { e_.check(pbsgpu_stream_write(s_, b.data(), b.size())); }
    void drain() {
        pbsgpu_chunk buf[256];
        for (;;) {
            uint64_t n = 0;
            e_.check(pbsgpu_stream_poll(s_, buf, 256, &n));
            if (!n) break;
            for (uint64_t i = 0; i < n; i++) {
                PayloadChunk c; c.end_off = buf[i].end_off; std::memcpy(c.digest, buf[i].digest, 32);
                c.known = (buf[i].flags & PBSGPU_CHUNK_KNOWN) != 0;
                index_.push_back(c);
                if (upload_ && !c.known) pending_.push_back(index_.size() - 1);
            }
        }
        // blob k belongs to the k-th new record: ask only for blobs whose records are here already
        uint64_t lens[256];
        while (!pending_.empty()) {
            uint64_t n = 0;
            const uint64_t cap = pending_.size() < 256 ? pending_.size() : 256;
            e_.check(pbsgpu_stream_poll_blobs(s_, blob_buf_.data(), blob_buf_.size(), lens, cap, &n));
            if (!n) break;
            const uint8_t *b = blob_buf_.data();
            for (uint64_t i = 0; i < n; b += lens[i], i++) {
                upload_(index_[pending_.front()].digest, b, lens[i]);
                pending_.pop_front();
            }
        }
        uint64_t h[256];
        for (uint64_t n = 1; n && !hashed_.empty();) {
            e_.check(pbsgpu_stream_poll_hashes(s_, h, 256, &n));
            for (uint64_t i = 0; i < n; i++) { backed_hashes_[hashed_.front()] = h[i]; hashed_.pop_front(); }
        }
    }
    Engine &e_;
    pbsgpu_stream *s_ = nullptr;
    bool suggest_, finished_ = false;
    UploadBlob upload_;
    bool hash_;
    std::vector<uint8_t> blob_buf_;
    std::vector<PayloadChunk> index_;
    std::deque<size_t> pending_;          // index_ positions of new chunks whose blob has not come back yet
    std::deque<std::string> hashed_;      // paths whose hash has not come back yet
    std::map<std::string, uint64_t> backed_hashes_;
};

// ---- disk images: a fixed index (<name>.img.fidx) ---------------------------------------------------------------------
// The image is cut at every multiple of `chunk_size` (upstream writes 4 MiB).  WriteSlice takes the next bytes of the
// image (HOST or DEVICE memory); every slice but the last is a multiple of chunk_size.  Each chunk is digested on the
// GPU (keyed with `crypt`) and probed against `known` (seed it with KnownSet::SeedFromFidx); with a blob mode
// (PBSGPU_BLOB_RAW .. _LZH, _LZL, _LZC), every new chunk's DataBlob goes to `upload_blob` (encrypted with `crypt`, IVs from
// getrandom).  Finish() renders the .fidx.
class FixedIndexWriter {
  public:
    FixedIndexWriter(Engine &e, uint32_t chunk_size, KnownSet *known, int blob_mode = PBSGPU_BLOB_NONE,
                     UploadBlob upload_blob = nullptr, const CryptConfig *crypt = nullptr)
        : e_(e), cs_(chunk_size), known_(known), mode_(blob_mode), upload_(std::move(upload_blob)), crypt_(crypt) {
        if ((mode_ != PBSGPU_BLOB_NONE) != (upload_ != nullptr))
            throw Error(PBSGPU_EINVAL, "transfer: a blob mode and an upload_blob callback go together");
    }
    void WriteSlice(const uint8_t *data, uint64_t len) {
        if (len == 0) return;
        if (ended_) throw Error(PBSGPU_EINVAL, "transfer: the image's last slice ended inside a chunk; no slice may follow it");
        const uint64_t off = 0, n = (len + cs_ - 1) / cs_;
        std::vector<pbsgpu_chunk> out(n);
        uint64_t got = 0;
        pbsgpu_batch_opts o = {sizeof(pbsgpu_batch_opts), 0, known_ ? known_->handle() : nullptr, nullptr, nullptr, 0,
                               nullptr, crypt_ ? crypt_->handle() : nullptr, cs_};
        e_.check(pbsgpu_chunk_digest_batch_ex(e_.ctx(), nullptr, data, &off, &len, 1, &o, out.data(), n, &got));
        std::vector<uint64_t> boff, blen;
        std::vector<const uint8_t *> bdig;
        for (uint64_t i = 0; i < got; i++) {
            digests_.insert(digests_.end(), out[i].digest, out[i].digest + 32);
            known_flags_.push_back((out[i].flags & PBSGPU_CHUNK_KNOWN) != 0);
            if (!known_flags_.back()) { boff.push_back(i * cs_); blen.push_back(std::min<uint64_t>(cs_, len - i * cs_)); bdig.push_back(out[i].digest); }
        }
        if (upload_ && !boff.empty()) upload(data, boff, blen, bdig);
        size_ += len;
        ended_ = len % cs_ != 0;
    }
    // The image's .fidx (checksum on the GPU).
    std::vector<uint8_t> Finish(const uint8_t uuid[16] = nullptr, int64_t ctime = 0) {
        const uint8_t zero[16] = {};
        const uint64_t n = digests_.size() / 32;
        std::vector<uint8_t> img(pbsgpu_fidx_size(n));
        e_.check(pbsgpu_fidx_build(e_.ctx(), digests_.data(), n, size_, cs_, uuid ? uuid : zero, ctime, img.data(), img.size()));
        return img;
    }
    const std::vector<uint8_t> &Digests() const { return digests_; }   // 32 bytes per chunk, in image order
    const std::vector<bool> &Known() const { return known_flags_; }
    uint64_t Size() const { return size_; }

  private:
    void upload(const uint8_t *data, const std::vector<uint64_t> &off, const std::vector<uint64_t> &len,
                const std::vector<const uint8_t *> &dig) {
        const uint32_t n = (uint32_t)off.size();
        std::vector<uint64_t> out_off(n + 1, 0), out_len(n);
        for (uint32_t i = 0; i < n; i++)
            out_off[i + 1] = out_off[i] + (crypt_ ? pbsgpu_blob_size_enc(len[i]) : pbsgpu_blob_size(len[i]));
        std::vector<uint8_t> buf(out_off[n]);
        if (crypt_) {
            std::vector<uint8_t> iv(16ull * n);
            for (size_t k = 0; k < iv.size();) {
                const ssize_t r = getrandom(iv.data() + k, iv.size() - k, 0);
                if (r <= 0) throw Error(PBSGPU_EINVAL, "transfer: getrandom failed");
                k += (size_t)r;
            }
            e_.check(pbsgpu_blob_encode_batch_enc(e_.ctx(), crypt_->handle(), mode_, data, off.data(), len.data(), n, iv.data(),
                                                  buf.data(), out_off.data(), out_len.data(), nullptr));
        } else if (mode_ == PBSGPU_BLOB_RAW) {
            e_.check(pbsgpu_blob_encode_batch(e_.ctx(), data, off.data(), len.data(), n, buf.data(), out_off.data(), nullptr));
            for (uint32_t i = 0; i < n; i++) out_len[i] = out_off[i + 1] - out_off[i];
        } else {
            auto fn = mode_ == PBSGPU_BLOB_Z ? pbsgpu_blob_encode_batch_z : mode_ == PBSGPU_BLOB_LZ ? pbsgpu_blob_encode_batch_lz
                    : mode_ == PBSGPU_BLOB_LZE ? pbsgpu_blob_encode_batch_lze : mode_ == PBSGPU_BLOB_LZH ? pbsgpu_blob_encode_batch_lzh
                    : mode_ == PBSGPU_BLOB_LZL ? pbsgpu_blob_encode_batch_lzl : mode_ == PBSGPU_BLOB_LZC ? pbsgpu_blob_encode_batch_lzc
                    : nullptr;
            if (!fn) throw Error(PBSGPU_EINVAL, "transfer: unknown blob mode " + std::to_string(mode_));
            e_.check(fn(e_.ctx(), data, off.data(), len.data(), n, buf.data(), out_off.data(), out_len.data(), nullptr));
        }
        for (uint32_t i = 0; i < n; i++) upload_(dig[i], buf.data() + out_off[i], out_len[i]);
    }
    Engine &e_;
    uint32_t cs_;
    KnownSet *known_;
    int mode_;
    UploadBlob upload_;
    const CryptConfig *crypt_;
    std::vector<uint8_t> digests_;
    std::vector<bool> known_flags_;
    uint64_t size_ = 0;
    bool ended_ = false;
};

}  // namespace transfer
}  // namespace pbsgpu
