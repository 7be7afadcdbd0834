// pbs_plus_b200/csrc/capi_blob.cu -- DataBlobs (pbsgpu_blob_*): the format, the encoder of new chunks (zstd frames on the
// device, optional AES-256-GCM, K6's CRC) and the batched decode and verify of stored ones.  All blocking calls
// (host.hpp, Blocking).
#include <algorithm>
#include <cstring>

#include "host.hpp"

using namespace pbsgpu;

// ---------------------------------------------------------------------------
// the format (upstream pbs-datastore data_blob.rs): magic[8] | crc32 LE over the payload | payload, with the IV and the
// GCM tag in front of the payload of an encrypted blob
// ---------------------------------------------------------------------------
// the magics in K13's order: a blob's kind is its index here, 2 * encrypted + compressed
static const uint8_t BLOB_MAGICS[4][8] = {
    {66, 171, 56, 7, 190, 131, 112, 161},                     // uncompressed
    {49, 185, 88, 66, 111, 182, 163, 127},                    // zstd compressed
    {0x7b, 0x67, 0x85, 0xbe, 0x22, 0x2d, 0x4c, 0xf0},         // encrypted
    {0xe6, 0x59, 0x1b, 0xbf, 0x0b, 0xbf, 0xd8, 0x0b}};        // zstd compressed, encrypted

static void blob_header(const uint8_t magic[8], uint32_t crc, uint8_t *out) {
    memcpy(out, magic, 8);
    for (int i = 0; i < 4; i++) out[8 + i] = (uint8_t)(crc >> (8 * i));
}
extern "C" void pbsgpu_blob_header(uint32_t crc, uint8_t out[12]) { blob_header(BLOB_MAGICS[0], crc, out); }
extern "C" uint64_t pbsgpu_blob_size(uint64_t payload_len) { return payload_len + 12; }
extern "C" uint64_t pbsgpu_blob_size_enc(uint64_t payload_len) { return payload_len + 44; }

// Which DataBlob encoder a call is: uncompressed only, RLE / raw frames (_z), with the match stage (_lz), with the match
// and entropy stages (_lze), with Huffman literals over every byte value (_lzh), _lzh with long-distance matches
// across the whole chunk (_lzl), and _lzh with K16's hash-chain search over the whole chunk and lazy parse (_lzc).
enum class BlobMode { raw, z, lz, lze, lzh, lzl, lzc };
// the encoders by their PBSGPU_BLOB_* value (PBSGPU_BLOB_RAW ..); values 6, 8 and 9 are not assigned
static bool blob_mode_of(int mode, BlobMode *m) {
    static const BlobMode modes[] = {BlobMode::raw, BlobMode::z, BlobMode::lz, BlobMode::lze, BlobMode::lzh};
    if (mode >= PBSGPU_BLOB_RAW && mode <= PBSGPU_BLOB_LZH) { *m = modes[mode - PBSGPU_BLOB_RAW]; return true; }
    if (mode == PBSGPU_BLOB_LZL) { *m = BlobMode::lzl; return true; }
    if (mode == PBSGPU_BLOB_LZC) { *m = BlobMode::lzc; return true; }
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

// K16 (lzc): the passes of whole chunks (at most CH_PASS_BYTES, or one longer chunk) that hold blocks of the match
// stage's list (zfirst[i]: chunk i's first; vfirst, vpos: zchain.cuh's numbering, vpos uploaded here); per pass the chain
// search, then parse(args, scratch) enqueues K16c and the encoders.  The scratch is sized once for the largest pass.
template <class Parse>
static int chain_passes(Blocking &b, const uint8_t *dbase, const uint64_t *d_off, const uint64_t *d_len, uint32_t n,
                        const std::vector<uint64_t> &vfirst, const std::vector<uint64_t> &zfirst,
                        const std::vector<uint64_t> &vpos, const uint64_t *d_zsrc, const uint32_t *d_zsize, Parse parse) {
    pbsgpu_ctx *ctx = b.ctx;
    std::vector<uint32_t> pass_c0;
    for (uint32_t i = 0; i < n; i++)
        if (pass_c0.empty() || vfirst[i + 1] - vfirst[pass_c0.back()] > CH_PASS_BYTES) pass_c0.push_back(i);
    pass_c0.push_back(n);
    size_t scratch_bytes = 0;
    for (size_t p = 0; p + 1 < pass_c0.size(); p++)
        if (zfirst[pass_c0[p + 1]] > zfirst[pass_c0[p]])
            scratch_bytes = std::max(scratch_bytes, chain_scratch_bytes(vfirst[pass_c0[p + 1]] - vfirst[pass_c0[p]]));
    uint64_t *d_vfirst = b.upload(vfirst.data(), n + 1), *d_vpos = b.upload(vpos.data(), vpos.size());
    uint8_t *scratch = b.get<uint8_t>(scratch_bytes);
    if (!d_vfirst || !d_vpos || !scratch)
        return fail(ctx, PBSGPU_ENOMEM, "chain search scratch of %llu bytes failed", (unsigned long long)scratch_bytes);
    for (size_t p = 0; b.ok() && p + 1 < pass_c0.size(); p++) {
        const uint32_t c0 = pass_c0[p], c1 = pass_c0[p + 1];
        const ChainArgs a{dbase, d_off, d_len, d_vfirst, c0, c1, vfirst[c1] - vfirst[c0], vfirst[c0], d_zsrc, d_vpos, d_zsize,
                          zfirst[c0], zfirst[c1]};
        if (a.z1 == a.z0) continue;
        b.e = launch_chain_search(a, scratch, b.st);
        parse(a, (void *)scratch);
    }
    return PBSGPU_OK;
}

// Compressed form: a blob's payload is a zstd frame when that is smaller than the raw bytes (upstream
// `DataBlob::encode` keeps the compressed form only then).  The frame is built on the device (zframe.cu, zlz.cu,
// zent.cu): a 128 KiB block of one repeated byte is an RLE_Block (K8a decides); with lz / lze / lzh every other block
// goes through the match stage (K9; lze and lzh add the entropy stage, K10, lzh with its full-alphabet flag) and is a
// Compressed_Block when that is smaller than the block; the rest are Raw_Blocks.  Marks those blobs in comp[] and points
// their payloads (at[i], plen[i]) to their frames in the frame stage *frames, a block of `b`.
static int zstd_frames(Blocking &b, const uint8_t *dbase, const uint64_t *off, const uint64_t *len, uint32_t n, BlobMode mode,
                       std::vector<uint8_t> &comp, std::vector<const uint8_t *> &at, std::vector<uint64_t> &plen,
                       const uint8_t **frames) {
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
    // K10) into slots nz + y, and each such block keeps the smaller content, K9's on ties.  With lzc, K16 is the parse
    // instead of K9a, per pass of whole chunks (CH_PASS_BYTES, or one longer chunk).
    const bool lzc = mode == BlobMode::lzc;
    const bool ent = mode == BlobMode::lze || mode == BlobMode::lzh || mode == BlobMode::lzl || lzc, lz = mode == BlobMode::lz || ent;
    const bool full = mode == BlobMode::lzh || mode == BlobMode::lzl || lzc;
    std::vector<uint32_t> info;
    std::vector<uint64_t> slot_of;   // the slot of block z's content
    const uint8_t *slots = nullptr;
    if (lz) {
        std::vector<uint64_t> zsrc;
        std::vector<uint32_t> zsize;
        std::vector<int64_t> zof(n_blocks, -1);
        std::vector<uint64_t> zfirst(n + 1), vfirst(n + 1), vpos;   // lzc: K16's numbering (zchain.cuh, ChainArgs)
        for (uint32_t i = 0; i < n; i++) {
            zfirst[i] = zsrc.size();
            vfirst[i + 1] = vfirst[i] + len[i];
            for (uint64_t k = 0; k < blk_first[i + 1] - blk_first[i]; k++)
                if (!(flags[blk_first[i] + k] & 0x100u)) {
                    zof[blk_first[i] + k] = (int64_t)zsrc.size();
                    zsrc.push_back(off[i] + k * ZFRAME_BLOCK); zsize.push_back(block_size(i, k));
                    if (lzc) vpos.push_back(vfirst[i] + k * ZFRAME_BLOCK);
                }
        }
        zfirst[n] = zsrc.size();
        const uint64_t nz = zsrc.size();
        std::vector<uint32_t> span_z, span_first;
        std::vector<uint64_t> spans;
        if (mode == BlobMode::lzl && nz)
            if (int rc = ldm_spans_of(b, dbase, off, len, n, blk_first, zof, span_z, span_first, spans)) return rc;
        const uint64_t ny = span_z.size();
        for (uint64_t y = 0; y < ny; y++) { zsrc.push_back(zsrc[span_z[y]]); zsize.push_back(zsize[span_z[y]]); }
        if (nz) {
            if (int rc = pbsgpu_upload_table_once(ctx, &ctx->d_lz_tab, sizeof(LzTables), lz_fill_tables_host)) return rc;
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
            // K9b and K10 over blocks [f, f + pn), parsed into the pass scratch
            auto encode = [&](uint64_t f, uint32_t pn) {
                if (b.ok()) b.e = launch_lz_encode((const LzTables *)ctx->d_lz_tab, f, pn, d_slots, d_seqs, d_nseq, d_nlit, d_info, b.st);
                if (b.ok() && d_ent)
                    b.e = launch_ent_encode((const LzTables *)ctx->d_lz_tab, d_zsize, f, pn, d_slots, d_seqs, d_nseq, d_nlit,
                                            d_info, d_ent, full, b.st);
            };
            // the blocks [0, nz), then the span blocks [nz, nz + ny), each list in passes of its own
            auto passes = [&](uint64_t lo, uint64_t hi, bool span_parse) {
                for (uint64_t f = lo; b.ok() && f < hi; f += LZ_PASS_BLOCKS) {
                    const uint32_t pn = (uint32_t)std::min<uint64_t>(LZ_PASS_BLOCKS, hi - f);
                    b.e = span_parse ? launch_lz_parse_spans(dbase, d_zsrc, d_zsize, f, pn, d_slots, d_seqs, d_nseq, d_nlit,
                                                             d_spans, d_span_first, nz, b.st)
                                     : launch_lz_parse(dbase, d_zsrc, d_zsize, f, pn, d_slots, d_seqs, d_nseq, d_nlit, b.st);
                    encode(f, pn);
                }
            };
            if (lzc) {   // K16c and the encoders per pass, LZ_PASS_BLOCKS blocks at a time
                auto parse = [&](const ChainArgs &a, void *scratch) {
                    for (uint64_t f = a.z0; b.ok() && f < a.z1; f += LZ_PASS_BLOCKS) {
                        const uint32_t pn = (uint32_t)std::min<uint64_t>(LZ_PASS_BLOCKS, a.z1 - f);
                        b.e = launch_chain_parse(a, scratch, f, pn, d_slots, d_seqs, d_nseq, d_nlit, b.st);
                        encode(f, pn);
                    }
                };
                if (int rc = chain_passes(b, dbase, d_off, d_len, n, vfirst, zfirst, vpos, d_zsrc, d_zsize, parse)) return rc;
            } else {
                passes(0, nz, false);
            }
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
        comp[i] = 1; plen[i] = fl;
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
    for (uint32_t i = 0, k = 0; i < n; i++)
        if (comp[i]) at[i] = stage + foff[k++];
    *frames = stage;
    return b.finish("zstd frame emit");
}

// K11's device buffers, sized once for a call's largest pass of n messages and segs segments
struct GcmBufs {
    GcmMsg *msg;
    uint64_t *seg_first;
    uint8_t *part, *tags;
    bool get(Blocking &b, uint64_t n, uint64_t segs) {
        msg = b.get<GcmMsg>(n); seg_first = b.get<uint64_t>(n + 1);
        part = b.get<uint8_t>(segs * 16 + 16); tags = b.get<uint8_t>(16 * n);
        return msg && seg_first && part && tags;
    }
};

// K11 over the messages msg[] (src, dst and len set) with the 16-byte IVs iv[k]: J0 and E_K(J0) of every message from its
// IV, the segment prefix, the launch (encrypt or decrypt) and the tags back into tags[16 k].  Waits for the stream.
static int gcm_run(Blocking &b, const pbsgpu_crypt *crypt, const GcmBufs &d, std::vector<GcmMsg> &msg,
                   const std::vector<const uint8_t *> &iv, bool decrypt, std::vector<uint8_t> &tags) {
    const uint32_t ne = (uint32_t)msg.size();
    std::vector<uint64_t> seg_first(ne + 1, 0);
    for (uint32_t k = 0; k < ne; k++) {
        gcm_j0_host(crypt->tab.data(), iv[k], msg[k].j0);
        gcm_encrypt_block_host(crypt->tab.data(), msg[k].j0, msg[k].ej0);
        seg_first[k + 1] = seg_first[k] + gcm_segments(msg[k].len);
    }
    tags.resize(16ull * ne);
    if (b.ok()) b.e = cudaMemcpyAsync(d.msg, msg.data(), ne * sizeof(GcmMsg), cudaMemcpyHostToDevice, b.st);
    if (b.ok()) b.e = cudaMemcpyAsync(d.seg_first, seg_first.data(), (ne + 1) * 8ull, cudaMemcpyHostToDevice, b.st);
    if (b.ok()) b.e = launch_gcm(d.msg, d.seg_first, ne, seg_first[ne], crypt->d_tab, d.part, d.tags, b.ctx->sm_count, b.st, decrypt);
    if (b.ok()) b.e = cudaMemcpyAsync(tags.data(), d.tags, 16ull * ne, cudaMemcpyDeviceToHost, b.st);
    return b.finish(decrypt ? "blob decryption" : "aes-256-gcm");
}

// ---------------------------------------------------------------------------
// f3: complete DataBlobs for the NEW chunks of a batch in one call (uploaded by POST /dynamic_chunk, reference
// internal/server/backup/log_cleanup.go:19-31)
// ---------------------------------------------------------------------------
// The payload is the zstd frame where that is smaller (zstd_frames) unless `mode` is raw, else the chunk.  With crypt, K11
// encrypts each payload from where it lies (the caller's device memory, the H2D stage or the frame stage) into a
// ciphertext stage, and that is the payload.  K6 takes the CRCs on the device, one launch per place the payloads lie in.
// Payload bytes are copied once straight into their place behind the header: device -> host for resident data, frames
// and ciphertext, host -> host for a plain raw payload of a host `base`.
int pbsgpu_blob_encode(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, int mode, const uint8_t *iv, const void *base,
                       const uint64_t *off, const uint64_t *len, uint32_t n, uint8_t *out, const uint64_t *out_off,
                       uint64_t *out_len, uint32_t *crc_out) {
    Guard g(ctx);
    BlobMode bm;
    if (!blob_mode_of(mode, &bm)) return fail(ctx, PBSGPU_EINVAL, "unknown blob mode %d", mode);
    if (n == 0) return PBSGPU_OK;
    const unsigned max_log2 = crypt ? 36 : 40;   // plain raw blobs have no limit
    for (uint32_t i = 0; (crypt || bm != BlobMode::raw) && i < n; i++)
        if (len[i] >= (1ull << max_log2)) return fail(ctx, PBSGPU_EINVAL, "blob %u longer than 2^%u bytes", i, max_log2);
    for (uint32_t i = 0; bm == BlobMode::lzc && i < n; i++)   // K16 numbers a pass's positions in 32 bits
        if (len[i] >= (1ull << 32)) return fail(ctx, PBSGPU_EINVAL, "lzc blob %u longer than 2^32 - 1 bytes", i);
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase, *frames = nullptr;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    // payload i: plen[i] bytes at the device address at[i], the chunk unless zstd_frames makes a smaller frame (comp[i])
    std::vector<uint8_t> comp(n, 0);
    std::vector<const uint8_t *> at(n);
    std::vector<uint64_t> plen(len, len + n);
    for (uint32_t i = 0; i < n; i++) at[i] = dbase + off[i];
    if (bm != BlobMode::raw)
        if (int rc = zstd_frames(b, dbase, off, len, n, bm, comp, at, plen, &frames)) return rc;
    std::vector<uint8_t> tags;
    uint8_t *ct = nullptr;
    if (crypt) {   // K11: payload i -> the ciphertext stage ct, 16 B aligned
        uint64_t bytes = 0, segs = 0;
        for (uint64_t l : plen) { bytes += (l + 15) & ~15ull; segs += gcm_segments(l); }
        ct = b.get<uint8_t>(bytes + 16);
        if (!ct) return fail(ctx, PBSGPU_ENOMEM, "ciphertext staging of %llu bytes failed", (unsigned long long)bytes);
        GcmBufs d;
        if (!d.get(b, n, segs)) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
        std::vector<GcmMsg> msg(n);
        std::vector<const uint8_t *> ivs(n);
        for (uint64_t i = 0, c = 0; i < n; i++) {
            msg[i] = {(uint64_t)(uintptr_t)at[i], (uint64_t)(uintptr_t)(ct + c), plen[i], {}, {}};
            ivs[i] = iv + 16 * i;
            at[i] = ct + c;
            c += (plen[i] + 15) & ~15ull;
        }
        if (int rc = gcm_run(b, crypt, d, msg, ivs, false, tags)) return rc;
    }
    // K6, one enqueue per place the payloads lie in: the ciphertext stage, or the frame stage and the input.  d_crc[r] is
    // the CRC of blob pick[r].
    uint32_t *d_crc = b.get<uint32_t>(n);
    if (!d_crc) return fail(ctx, PBSGPU_ENOMEM, "device allocation failed");
    std::vector<uint32_t> pick;
    auto crc_from = [&](const uint8_t *src, int want_comp) {   // the payloads in src with comp[i] == want_comp (< 0: all)
        std::vector<uint64_t> o, l;
        const size_t r0 = pick.size();
        for (uint32_t i = 0; i < n; i++)
            if (want_comp < 0 || comp[i] == want_comp) { pick.push_back(i); o.push_back(at[i] - src); l.push_back(plen[i]); }
        return o.empty() ? PBSGPU_OK : pbsgpu_crc32_enqueue(b, src, o.data(), l.data(), (uint32_t)o.size(), d_crc + r0);
    };
    if (int rc = crypt ? crc_from(ct, -1) : crc_from(frames, 1)) return rc;
    if (!crypt)
        if (int rc = crc_from(dbase, 0)) return rc;
    std::vector<uint32_t> crc_r(n), crc(n);
    if (b.ok()) b.e = cudaMemcpyAsync(crc_r.data(), d_crc, n * 4ull, cudaMemcpyDeviceToHost, b.st);
    if (int rc = b.finish("blob crc")) return rc;
    for (uint32_t r = 0; r < n; r++) crc[pick[r]] = crc_r[r];
    // assemble in the caller's memory
    const bool staged = dbase != (const uint8_t *)base;
    const uint64_t hs = crypt ? 44 : 12;
    cudaError_t e = cudaSuccess;
    for (uint32_t i = 0; i < n && e == cudaSuccess; i++) {
        uint8_t *blob = out + out_off[i];
        blob_header(BLOB_MAGICS[2 * (crypt != nullptr) + comp[i]], crc[i], blob);
        if (crypt) {
            memcpy(blob + 12, iv + 16ull * i, 16);
            memcpy(blob + 28, tags.data() + 16ull * i, 16);
        }
        if (out_len) out_len[i] = hs + plen[i];
        if (plen[i] == 0) continue;
        if (!crypt && !comp[i] && staged) memcpy(blob + hs, (const uint8_t *)base + off[i], plen[i]);
        else e = cudaMemcpyAsync(blob + hs, at[i], plen[i], cudaMemcpyDeviceToHost, ctx->copy_stream);
    }
    if (int rc = pbsgpu_finish(ctx, ctx->copy_stream, e, "blob assembly copy")) return rc;
    if (crc_out) memcpy(crc_out, crc.data(), (size_t)n * 4);
    return PBSGPU_OK;
}

// the checks of the plain encoders; pbsgpu_blob_encode_batch (PBSGPU_BLOB_RAW) has no out_len
static int blob_encode_plain(pbsgpu_ctx *ctx, int mode, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                             uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || (n && (!off || !len || !out || !out_off || (mode != PBSGPU_BLOB_RAW && !out_len) || !base))) return PBSGPU_EINVAL;
    return pbsgpu_blob_encode(ctx, nullptr, mode, nullptr, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                        uint8_t *out, const uint64_t *out_off, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_RAW, base, off, len, n, out, out_off, nullptr, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_z(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                          uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_Z, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lz(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                           uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_LZ, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lze(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_LZE, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lzh(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_LZH, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lzl(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_LZL, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_lzc(pbsgpu_ctx *ctx, const void *base, const uint64_t *off, const uint64_t *len, uint32_t n,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    return blob_encode_plain(ctx, PBSGPU_BLOB_LZC, base, off, len, n, out, out_off, out_len, crc_out);
}

extern "C" int pbsgpu_blob_encode_batch_enc(pbsgpu_ctx *ctx, const pbsgpu_crypt *crypt, int mode, const void *base,
                                            const uint64_t *off, const uint64_t *len, uint32_t n, const uint8_t *iv,
                                            uint8_t *out, const uint64_t *out_off, uint64_t *out_len, uint32_t *crc_out) {
    if (!ctx || !crypt || crypt->ctx != ctx || (n && (!off || !len || !iv || !out || !out_off || !out_len || !base)))
        return PBSGPU_EINVAL;
    return pbsgpu_blob_encode(ctx, crypt, mode, iv, base, off, len, n, out, out_off, out_len, crc_out);
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
    if (int rc = pbsgpu_upload_table_once(ctx, &ctx->d_zdec_tab, sizeof(ZdecTables), zdec_fill_tables_host)) return rc;
    const bool out_dev = out && pbsgpu_is_device_ptr(out), want_sha = digest || digest_out;
    Blocking b(ctx, ctx->streams[0]);
    const uint8_t *dbase;
    if (int rc = b.stage(base, off, len, n, &dbase)) return rc;
    // kind[i]: the magic's index in BLOB_MAGICS (K13's order), -1 for an unknown magic or a blob shorter than its header;
    // without crypt every blob is left to K13 (0).  heads: the first ZDEC_HEAD bytes of every blob.
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
    // encrypt mode: the plaintext stage and K11's buffers, for the largest pass
    uint8_t *stage = nullptr, *d_shead = nullptr;
    uint64_t *d_sat = nullptr;
    uint32_t *d_csub = nullptr;
    GcmBufs gcm;
    if (crypt) {
        stage = b.get<uint8_t>(stage_max + 16); d_shead = b.get<uint8_t>(blobs_max * 16);
        d_sat = b.get<uint64_t>(blobs_max); d_csub = b.get<uint32_t>(blobs_max);
        if (!gcm.get(b, blobs_max, segs_max) || !stage || !d_shead || !d_sat || !d_csub)
            return fail(ctx, PBSGPU_ENOMEM, "decryption stage (%llu bytes) failed", (unsigned long long)stage_max);
    }
    std::vector<ZdecBlob> zb(blobs_max);
    std::vector<uint64_t> at(blobs_max), sat(blobs_max);   // chunk k of the pass at pass base + at[k]; its plaintext blob at stage + sat[k]
    std::vector<ChunkRef> refs(blobs_max);
    std::vector<uint32_t> ref_blob(blobs_max), list(blobs_max), csub(blobs_max);
    std::vector<int32_t> st(blobs_max);
    std::vector<uint8_t> dig(blobs_max * 32), tags, shead;
    std::vector<GcmMsg> msg;
    std::vector<const uint8_t *> ivs;
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
        msg.clear(); ivs.clear(); list.clear();
        for (uint32_t k = 0; crypt && k < pn; k++) {
            const uint32_t i = i0 + k;
            if (kind[i] < 2 || status[i] != PBSGPU_DEC_OK) continue;
            msg.push_back({(uint64_t)(uintptr_t)(dbase + off[i] + ZDEC_HEAD), (uint64_t)(uintptr_t)(stage + sat[k] + 16), ct[i],
                           {}, {}});
            ivs.push_back(heads.data() + (size_t)ZDEC_HEAD * i + 12);
            list.push_back(k);
        }
        if (!msg.empty()) {
            if (int rc = gcm_run(b, crypt, gcm, msg, ivs, true, tags)) return rc;
            for (uint32_t r = 0; r < msg.size(); r++) {
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
            const unsigned long long hn = nr;
            if (b.ok()) b.e = cudaMemcpyAsync(d_refs, refs.data(), nr * sizeof(ChunkRef), cudaMemcpyHostToDevice, b.st);
            if (b.ok()) b.e = cudaMemcpyAsync(d_nref, &hn, sizeof hn, cudaMemcpyHostToDevice, b.st);
            pbsgpu_sha256_enqueue(b, pbase, d_refs, d_nref, nr, keyed ? pbsgpu_crypt_id_key(crypt) : nullptr, d_dig);
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
