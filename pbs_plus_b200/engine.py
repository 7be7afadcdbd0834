"""Host-side front end of the H100 chunk + digest + probe engine.

Thin, allocation-free wrappers over the C ABI (include/pbsgpu.h).  Device memory
comes from the caller (e.g. a torch CUDA tensor -- torch is plumbing only) or the
library stages host memory itself.  No CPU fallback: everything below runs the
sm_90a kernels in pbs_plus_b200/csrc/.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Sequence

import numpy as np

from . import _lib
from ._lib import BLOB_MODES, CHUNK_DTYPE, CHUNK_KNOWN, BatchOptsFixed, Cfg, Corpus, DevInfo, PbsGpuError, Timing


def _ptr(x) -> int:
    """Raw address of a torch tensor / numpy array / int."""
    if isinstance(x, int):
        return x
    if hasattr(x, "data_ptr"):
        return int(x.data_ptr())
    if isinstance(x, np.ndarray):
        return int(x.ctypes.data)
    if isinstance(x, (bytes, bytearray, memoryview)):
        return int(np.frombuffer(x, dtype=np.uint8).ctypes.data)
    raise TypeError(f"cannot take the address of {type(x)}")


def _cfg_ref(cfg: Cfg | None):
    return C.byref(cfg) if cfg is not None else None


def _offsets(sizes) -> tuple[np.ndarray, int]:
    """Ranges of `sizes` laid back to back -> (exclusive offsets u64[n], total)."""
    sizes = np.asarray(sizes, dtype=np.uint64)
    off = np.zeros(len(sizes), dtype=np.uint64)
    if len(sizes):
        off[1:] = np.cumsum(sizes)[:-1]
    return off, int(sizes.sum())


def _pack(arrays) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Host streams in one buffer, each starting 256-byte aligned -> (buf, off u64[n], len u64[n])."""
    arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in arrays]
    off, total = _offsets([(len(a) + 255) & ~255 for a in arrs])
    buf = np.zeros(max(total, 1), dtype=np.uint8)
    for a, o in zip(arrs, off):
        buf[int(o): int(o) + len(a)] = a
    return buf, off, np.array([len(a) for a in arrs], dtype=np.uint64)


def _join(items) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """`bytes`-like items back to back, unpadded -> (base, off u64[n], len u64[n]); the base of no items is b"\\0"."""
    lens = np.array([len(b) for b in items], dtype=np.uint64)
    off, _ = _offsets(lens)
    return np.frombuffer(b"".join(bytes(b) for b in items) or b"\0", dtype=np.uint8), off, lens


def _split(buf, off, length, keep=None) -> list:
    """buf[off[i]:off[i] + length[i]] per range: `bytes` from a numpy buffer, a view of a tensor; None where keep[i] is
    false."""
    views = [buf[int(a): int(a) + int(n)] if keep is None or keep[i] else None
             for i, (a, n) in enumerate(zip(off, length))]
    return [v.tobytes() if isinstance(v, np.ndarray) else v for v in views]


def _deflate_layout(l: np.ndarray, more):
    """Output room of n raw Deflate streams -> (out_off u64[n] spaced by deflate_bound, total bytes, more u8[n] or
    None)."""
    off, total = _offsets([deflate_bound(int(x)) for x in l])
    m = None if more is None else np.ascontiguousarray(more, dtype=np.uint8)
    if m is not None and m.shape != l.shape:
        raise ValueError("more must hold one flag per range")
    return off, total, m


def _digests(digests, per: str, n: int | None = None) -> np.ndarray:
    """Digests as `bytes` or an array, 32 bytes per item (n items, or any number) -> flat u8; `per` ends the error."""
    d = np.ascontiguousarray(np.frombuffer(bytes(digests), dtype=np.uint8) if isinstance(digests, (bytes, bytearray))
                             else np.asarray(digests, dtype=np.uint8)).reshape(-1)
    if d.size != 32 * (d.size // 32 if n is None else n):
        raise ValueError(f"digests must hold 32 bytes {per}")
    return d


def make_config(avg_bytes: int, table: np.ndarray | None = None) -> Cfg:
    """Chunker parameters; replaces buzhash.NewConfig (reference commit.go:302-305). avg in BYTES."""
    cfg = Cfg()
    tp = None
    if table is not None:
        table = np.ascontiguousarray(table, dtype=np.uint32)
        if table.shape != (256,):
            raise ValueError("table must hold 256 u32 entries")
        tp = table.ctypes.data_as(C.POINTER(C.c_uint32))
    rc = _lib.lib().pbsgpu_config(int(avg_bytes), tp, C.byref(cfg))
    if rc:
        raise PbsGpuError(rc, f"invalid average chunk size {avg_bytes} (power of two in [256, 2^29] required)")
    return cfg


def default_table() -> np.ndarray:
    return np.ctypeslib.as_array(_lib.lib().pbsgpu_default_table(), shape=(256,)).copy()


def deflate_bound(n: int) -> int:
    """pbsgpu_deflate_bound: the bytes every raw Deflate stream of n bytes fits in."""
    return int(_lib.lib().pbsgpu_deflate_bound(n))


def crc32_combine(crc1: int, crc2: int, len2: int) -> int:
    """CRC-32 of A || B from CRC-32(A), CRC-32(B) and len(B) (pbsgpu_crc32_combine, host only)."""
    return int(_lib.lib().pbsgpu_crc32_combine(crc1, crc2, len2))


def zip_entry(name: bytes, mode: int, mtime: int, method: int = 0, crc: int = 0, comp_size: int = 0, size: int = 0,
              offset: int = 0) -> "_lib.ZipEntry":
    """A pbsgpu_zip_entry; the returned structure keeps `name` alive."""
    name = bytes(name)
    buf = C.create_string_buffer(name, len(name) or 1)
    e = _lib.ZipEntry(C.cast(buf, C.c_void_p), len(name), mode, mtime, method, crc, comp_size, size, offset)
    e._keep = buf
    return e


def _zip_record(fn, *args) -> bytes:
    need = fn(*args, None, 0)
    out = C.create_string_buffer(max(1, need))
    assert fn(*args, out, need) == need
    return out.raw[:need]


def zip_local_header(e) -> bytes:
    """The local file header of an entry (pbsgpu_zip_local_header)."""
    return _zip_record(_lib.lib().pbsgpu_zip_local_header, C.byref(e))


def zip_data_descriptor(e) -> bytes:
    """The data descriptor behind an entry's content; b"" for a directory (pbsgpu_zip_data_descriptor)."""
    return _zip_record(_lib.lib().pbsgpu_zip_data_descriptor, C.byref(e))


def zip_directory(entries, offset: int) -> bytes:
    """The central directory of `entries` at archive offset `offset`, with its end records (pbsgpu_zip_directory)."""
    arr = (_lib.ZipEntry * max(1, len(entries)))(*entries)
    return _zip_record(_lib.lib().pbsgpu_zip_directory, arr, len(entries), offset)


class Engine:
    """One context on one GPU (pbsgpu_open).  Raises if the device or the .so is missing."""

    def __init__(self, device: int = 0, profiling: bool = False):
        self._L = _lib.lib()
        h = C.c_void_p()
        rc = self._L.pbsgpu_open(device, C.byref(h))
        if rc:
            raise PbsGpuError(rc, "pbsgpu_open failed: no usable CUDA device (there is no CPU fallback)")
        self._h = h
        self.device = device
        if profiling:
            self.set_profiling(True)

    # -- plumbing ------------------------------------------------------------------
    def _ck(self, rc: int):
        if rc:
            raise PbsGpuError(rc, (self._L.pbsgpu_strerror(self._h) or b"").decode())

    def close(self):
        if getattr(self, "_h", None):
            self._L.pbsgpu_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _alloc(self, nbytes: int, out: str | None):
        """The output buffer of a call (at least one byte): numpy for "host", a torch CUDA tensor on this engine's
        device for "device", None for None."""
        if out == "host":
            return np.zeros(max(1, nbytes), dtype=np.uint8)
        if out == "device":
            import torch
            return torch.empty(max(1, nbytes), dtype=torch.uint8, device=f"cuda:{self.device}")
        return None

    def device_info(self) -> dict:
        d = DevInfo()
        self._ck(self._L.pbsgpu_device_info(self._h, C.byref(d)))
        return {"device": d.device, "sm_count": d.sm_count, "cc": (d.cc_major, d.cc_minor),
                "total_mem": d.total_mem, "free_mem": d.free_mem, "name": d.name.decode()}

    def partition_info(self) -> tuple[int, int]:
        """(SMs reserved for long-chunk kernels, SMs for the rest); (0, 0) if not partitioned."""
        a, b = C.c_int(), C.c_int()
        self._ck(self._L.pbsgpu_partition_info(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def scan_partition_sms(self) -> int:
        """SMs reserved for the front halves (K1 scan / sort / K2 resolve); 0 = shared with the bulk partition."""
        return int(self._L.pbsgpu_scan_partition_sms(self._h))

    def set_profiling(self, on: bool):
        self._ck(self._L.pbsgpu_set_profiling(self._h, 1 if on else 0))

    def set_kernel_variant(self, variant: int):
        """0 = tuned kernels, 1 = simple cross-check kernels (identical results)."""
        self._ck(self._L.pbsgpu_set_kernel_variant(self._h, variant))

    # -- a2+a3(+a4): batch ----------------------------------------------------------
    @staticmethod
    def _offlen(off: Sequence[int], length: Sequence[int]):
        o = np.ascontiguousarray(off, dtype=np.uint64)
        l = np.ascontiguousarray(length, dtype=np.uint64)
        if o.shape != l.shape or o.ndim != 1:
            raise ValueError("off/len must be 1-D and of equal length")
        return o, l

    @staticmethod
    def _chunk_cap(cfg: Cfg | None, l: np.ndarray, fixed_size: int = 0, forced=None) -> int:
        extra = 1 + (len(forced[0]) if forced is not None else 0)
        if fixed_size:
            return int(((l + np.uint64(fixed_size - 1)) // np.uint64(fixed_size)).sum()) + extra
        m = max(int(cfg.min), 65)
        return int((l // np.uint64(m)).sum()) + len(l) + extra

    @staticmethod
    def _opts(digest_set, forced, xxh3=None, crypt=None, fixed_size: int = 0):
        """pbsgpu_batch_opts; `forced` = (stream u32[], offset u64[]) suggested boundaries sorted by (stream, offset);
        `crypt` (a Crypt) = keyed digests of encrypt mode; `fixed_size` = fixed cuts instead of the chunker."""
        o = BatchOptsFixed()
        o.size = C.sizeof(BatchOptsFixed)
        o.set = digest_set._h if digest_set is not None else None
        o.crypt = crypt._h if crypt is not None else None
        o.fixed_size = int(fixed_size)
        keep = []
        if forced is not None:
            fs = np.ascontiguousarray(forced[0], dtype=np.uint32)
            fo = np.ascontiguousarray(forced[1], dtype=np.uint64)
            if fs.shape != fo.shape or fs.ndim != 1:
                raise ValueError("forced = (stream[], offset[]) of equal length")
            o.forced_stream, o.forced_off, o.n_forced = fs.ctypes.data, fo.ctypes.data, len(fs)
            keep += [fs, fo]
        if xxh3 is not None:
            o.stream_xxh3 = xxh3.ctypes.data
        return o, keep

    def chunk_digest_batch(self, cfg: Cfg | None, base, off, length, digest_set: "DigestSet | None" = None,
                           forced=None, crypt: "Crypt | None" = None, fixed_size: int = 0) -> np.ndarray:
        """stream -> chunks -> digests for n streams; `base` device (tensor/int) or host (numpy).
        Replaces n calls of writer.WriteEntryReader (reference commit.go:720).  `forced` = optional suggested
        boundaries (stream[], offset[]): file starts of a pxar payload stream (pxarfs.go:408-411).  `crypt`: keyed
        digests SHA-256(chunk || id_key) of encrypt mode, also for the set's probe + insert.  `fixed_size`: cut every
        stream at multiples of it instead (the chunks of a .fidx image; cfg may be None)."""
        o, l = self._offlen(off, length)
        cap = self._chunk_cap(cfg, l, fixed_size, forced)
        out = np.zeros(cap, dtype=CHUNK_DTYPE)
        n_out = C.c_uint64()
        keep = base  # keep the buffer alive for the duration of the call
        opts, _k = self._opts(digest_set, forced, crypt=crypt, fixed_size=fixed_size)
        self._ck(self._L.pbsgpu_chunk_digest_batch_ex(
            self._h, _cfg_ref(cfg), _ptr(keep), o.ctypes.data, l.ctypes.data, len(o), C.byref(opts), out.ctypes.data, cap,
            C.byref(n_out)))
        return out[: n_out.value]

    def chunk_digest_batch_xxh3(self, cfg: Cfg, base, off, length, digest_set: "DigestSet | None" = None,
                                crypt: "Crypt | None" = None):
        """chunk_digest_batch plus the XXH3-64 of every stream from the same staged bytes (f2: the per-file
        hash of emitBackedFile, reference commit.go:717-725).  Returns (chunks, xxh3[n] uint64)."""
        o, l = self._offlen(off, length)
        cap = self._chunk_cap(cfg, l)
        out = np.zeros(cap, dtype=CHUNK_DTYPE)
        hashes = np.zeros(len(o), dtype=np.uint64)
        n_out = C.c_uint64()
        opts, _k = self._opts(digest_set, None, hashes, crypt)
        self._ck(self._L.pbsgpu_chunk_digest_batch_ex(
            self._h, C.byref(cfg), _ptr(base), o.ctypes.data, l.ctypes.data, len(o), C.byref(opts), out.ctypes.data,
            cap, C.byref(n_out)))
        return out[: n_out.value], hashes

    def chunk_digest_streams(self, cfg: Cfg, streams: Iterable[np.ndarray], digest_set=None) -> np.ndarray:
        """Convenience for host streams that are separate arrays: packs them and calls the batch ABI."""
        buf, offs, lens = _pack(streams)
        return self.chunk_digest_batch(cfg, buf, offs, lens, digest_set)

    def submit(self, cfg: Cfg | None, base_dev, off, length, digest_set: "DigestSet | None" = None, forced=None,
               early_input: bool = False, crypt: "Crypt | None" = None, fixed_size: int = 0) -> "Job":
        """Asynchronous form; with `digest_set` the probe + insert runs as kernels on the job's stream (jobs sharing a
        set are ordered in submission order) and the KNOWN flags come back with the records.  `early_input`
        (PBSGPU_BATCH_EARLY_INPUT): the long chunks are copied aside so that Job.wait_input() gives the buffer back
        long before the records are ready.  `crypt`, `fixed_size`: as chunk_digest_batch."""
        o, l = self._offlen(off, length)
        h = C.c_void_p()
        opts, _k = self._opts(digest_set, forced, crypt=crypt, fixed_size=fixed_size)
        if early_input:
            opts.flags |= _lib.BATCH_EARLY_INPUT
        self._ck(self._L.pbsgpu_batch_submit_ex(self._h, _cfg_ref(cfg), _ptr(base_dev), o.ctypes.data, l.ctypes.data,
                                                len(o), C.byref(opts), C.byref(h)))
        return Job(self, h, self._chunk_cap(cfg, l, fixed_size, forced), base_dev)

    def scan_batch(self, cfg: Cfg, base_dev, off, length):
        """Boundaries only (a2).  Returns (ends, stream_first)."""
        o, l = self._offlen(off, length)
        cap = self._chunk_cap(cfg, l)
        ends = np.zeros(cap, dtype=np.uint64)
        first = np.zeros(len(o) + 1, dtype=np.uint64)
        n_out = C.c_uint64()
        self._ck(self._L.pbsgpu_scan_batch(self._h, C.byref(cfg), _ptr(base_dev), o.ctypes.data, l.ctypes.data,
                                           len(o), ends.ctypes.data, cap, first.ctypes.data, C.byref(n_out)))
        return ends[: n_out.value], first

    def sha256_batch(self, base, off, length) -> np.ndarray:
        """SHA-256 of n byte ranges (a3); returns (n, 32) uint8."""
        o, l = self._offlen(off, length)
        out = np.zeros((len(o), 32), dtype=np.uint8)
        self._ck(self._L.pbsgpu_sha256_batch(self._h, _ptr(base), o.ctypes.data, l.ctypes.data, len(o),
                                             out.ctypes.data))
        return out

    def sha256_keyed_batch(self, crypt: "Crypt", base, off, length) -> np.ndarray:
        """Encrypt mode's keyed digests SHA-256(range || id_key) of n byte ranges; returns (n, 32) uint8."""
        o, l = self._offlen(off, length)
        out = np.zeros((len(o), 32), dtype=np.uint8)
        self._ck(self._L.pbsgpu_sha256_keyed_batch(self._h, crypt._h, _ptr(base), o.ctypes.data, l.ctypes.data, len(o),
                                                   out.ctypes.data))
        return out

    # -- f2: per-file content hash of the commit walk ---------------------------------------------
    def xxh3_batch(self, base, off, length) -> np.ndarray:
        """XXH3-64 (seed 0) of n byte ranges (host or device base) on the GPU; uint64[n]."""
        o, l = self._offlen(off, length)
        out = np.zeros(len(o), dtype=np.uint64)
        self._ck(self._L.pbsgpu_xxh3_batch(self._h, _ptr(base), o.ctypes.data, l.ctypes.data, len(o), out.ctypes.data))
        return out

    # -- f3: DataBlob checksums --------------------------------------------------------------
    def crc32_batch(self, base, off, length) -> np.ndarray:
        """zlib-compatible CRC-32 of n byte ranges (host or device base) on the GPU."""
        o, l = self._offlen(off, length)
        out = np.zeros(len(o), dtype=np.uint32)
        self._ck(self._L.pbsgpu_crc32_batch(self._h, _ptr(base), o.ctypes.data, l.ctypes.data, len(o), out.ctypes.data))
        return out

    def deflate_batch(self, base, off, length, more=None, out: str = "host"):
        """Raw Deflate streams (RFC 1951) of n byte ranges (host or device base) on the GPU (pbsgpu_deflate_batch).
        more: per range, a later call continues the stream (its length a multiple of DEFLATE_SEGMENT).
        out: "host" -> list of bytes, "device" -> list of torch CUDA tensor views.  -> (streams, crc32 u32[n])"""
        return self._deflate(self._L.pbsgpu_deflate_batch, base, off, length, more, out)

    def deflate_batch_lzc(self, base, off, length, more=None, out: str = "host"):
        """deflate_batch with a hash-chain search and lazy parse in each segment (pbsgpu_deflate_batch_lzc): smaller
        streams, at a lower rate."""
        return self._deflate(self._L.pbsgpu_deflate_batch_lzc, base, off, length, more, out)

    def _deflate(self, fn, base, off, length, more, out):
        if out not in ("host", "device"):
            raise ValueError(f"out must be 'host' or 'device', not {out!r}")
        o, l = self._offlen(off, length)
        n = len(o)
        ooff, total, m = _deflate_layout(l, more)
        buf = self._alloc(total, out)
        olen = np.zeros(n, dtype=np.uint64)
        crc = np.zeros(n, dtype=np.uint32)
        self._ck(fn(self._h, _ptr(base), o.ctypes.data, l.ctypes.data, n, None if m is None else m.ctypes.data, _ptr(buf),
                    ooff.ctypes.data, olen.ctypes.data, crc.ctypes.data))
        return _split(buf, ooff, olen), crc

    def blob_encode_batch(self, base, off, length):
        """Complete uncompressed DataBlobs (magic | crc32 | payload) of n ranges -> (bytes buffer, blob_off[n+1], crc[n])."""
        o, l = self._offlen(off, length)
        out, boff, crc = self._blob_layout(l, 12)
        self._ck(self._L.pbsgpu_blob_encode_batch(self._h, _ptr(base), o.ctypes.data, l.ctypes.data, len(o),
                                                  out.ctypes.data if len(out) else None, boff.ctypes.data, crc.ctypes.data))
        return out, boff, crc

    def blob_encode_batch_z(self, base, off, length):
        """DataBlobs with a zstd payload where that is smaller (RLE / raw block frames, pbsgpu_blob_encode_batch_z)
        -> list of n `bytes` blobs, crc[n]."""
        return self._blob_encode_sized(self._L.pbsgpu_blob_encode_batch_z, base, off, length)

    def blob_encode_batch_lz(self, base, off, length):
        """blob_encode_batch_z with the match stage: blocks that are not constant become zstd Compressed_Blocks (greedy
        LZ77, raw literals, predefined FSE tables) where smaller (pbsgpu_blob_encode_batch_lz) -> list of n `bytes`
        blobs, crc[n]."""
        return self._blob_encode_sized(self._L.pbsgpu_blob_encode_batch_lz, base, off, length)

    def blob_encode_batch_lze(self, base, off, length):
        """blob_encode_batch_lz with zstd's entropy stage: each compressed block is the smaller of the _lz one and one
        with tables fitted to the block (FSE_Compressed_Mode sequences, Huffman literals) (pbsgpu_blob_encode_batch_lze)
        -> list of n `bytes` blobs, crc[n]."""
        return self._blob_encode_sized(self._L.pbsgpu_blob_encode_batch_lze, base, off, length)

    def blob_encode_batch_lzh(self, base, off, length):
        """blob_encode_batch_lze with Huffman literals whatever their largest value (the tree in the direct or the
        FSE-compressed weight form, the smaller one), so binary data gets entropy-coded literals too; every blob is at
        most its _lze blob (pbsgpu_blob_encode_batch_lzh) -> list of n `bytes` blobs, crc[n]."""
        return self._blob_encode_sized(self._L.pbsgpu_blob_encode_batch_lzh, base, off, length)

    def blob_encode_batch_lzl(self, base, off, length):
        """blob_encode_batch_lzh plus long-distance matches: repeats anywhere earlier in the same chunk (copies of a
        file, repeated pages), found by K12 and taken by the blocks they cross where that is smaller; every blob is at
        most its _lzh blob (pbsgpu_blob_encode_batch_lzl) -> list of n `bytes` blobs, crc[n]."""
        return self._blob_encode_sized(self._L.pbsgpu_blob_encode_batch_lzl, base, off, length)

    def blob_encode_batch_lzc(self, base, off, length):
        """blob_encode_batch_lzh with K16's match search: the longest of 16 hash-chain candidates anywhere up to 2^24 - 4
        bytes back in the chunk and a lazy parse, for smaller blobs of text-like data at more device time
        (pbsgpu_blob_encode_batch_lzc; ranges < 2^32 bytes) -> list of n `bytes` blobs, crc[n]."""
        return self._blob_encode_sized(self._L.pbsgpu_blob_encode_batch_lzc, base, off, length)

    @staticmethod
    def _blob_layout(l, head: int):
        """Room for n blobs back to back, each its uncompressed payload behind a `head`-byte header (12, or 44 encrypted)
        -> (out buffer, blob_off[n+1], crc[n])."""
        off, total = _offsets(l + np.uint64(head))
        return np.zeros(total, dtype=np.uint8), np.append(off, np.uint64(total)), np.zeros(len(l), dtype=np.uint32)

    def _blob_encode_sized(self, fn, base, off, length, head: int = 12):
        """Blobs whose sizes the encoder reports: fn(ctx, base, off, len, n, out, blob_off, blob_len, crc) -> list of n
        `bytes` blobs, crc[n]."""
        o, l = self._offlen(off, length)
        out, boff, crc = self._blob_layout(l, head)
        blen = np.zeros(len(o), dtype=np.uint64)
        self._ck(fn(self._h, _ptr(base), o.ctypes.data, l.ctypes.data, len(o), out.ctypes.data, boff.ctypes.data,
                    blen.ctypes.data, crc.ctypes.data))
        return _split(out, boff, blen), crc

    # -- f3, read side -------------------------------------------------------------------------
    def blob_decode_batch(self, blobs, chunk_len, digests=None, out: str | None = "host"):
        """Check, decode and verify unencrypted DataBlobs on the GPU (pbsgpu_blob_decode_batch).  `blobs` is a list of
        `bytes`, or (base, off[n], len[n]) with a host or device base; chunk_len[n] the expected chunk sizes (from the
        index); digests (n x 32 bytes, or None) the expected SHA-256s.  out: "host" (numpy), "device" (a torch CUDA
        tensor) or None (verify only: no decoded byte leaves the GPU).
        -> (status int32[n] (DEC_STATUS names them), data, digests u8[n, 32]); data is a list of n chunks (`bytes` for
        "host", tensor views for "device", None for blobs whose status is neither OK nor BAD_DIGEST), or None."""
        return self._blob_decode(lambda *a: self._L.pbsgpu_blob_decode_batch(self._h, *a), blobs, chunk_len, digests, out)

    def blob_decode_batch_enc(self, crypt: "Crypt", blobs, chunk_len, digests=None, out: str | None = "host"):
        """blob_decode_batch for encrypted and unencrypted DataBlobs (pbsgpu_blob_decode_batch_enc): encrypted blobs are
        decrypted with `crypt`'s key after their GCM tag verified (DEC_BAD_TAG otherwise), and their digests are keyed
        (SHA-256(chunk || id_key)), as in the index an encrypt-mode writer made; unencrypted blobs get plain digests."""
        return self._blob_decode(lambda *a: self._L.pbsgpu_blob_decode_batch_enc(self._h, crypt._h if crypt is not None else None, *a), blobs, chunk_len,
                                 digests, out)

    def _blob_decode(self, call, blobs, chunk_len, digests, out):
        if out not in ("host", "device", None):
            raise ValueError(f"out must be 'host', 'device' or None, not {out!r}")
        if isinstance(blobs, tuple):
            base, o, l = blobs
            o, l = self._offlen(o, l)
        else:
            base, o, l = _join(blobs)
        n = len(o)
        cl = np.ascontiguousarray(chunk_len, dtype=np.uint64)
        if cl.shape != (n,):
            raise ValueError("chunk_len must hold one size per blob")
        dg = None if digests is None else _digests(digests, "per blob", n)
        ooff, total = _offsets(cl)
        buf = self._alloc(total, out)
        status = np.zeros(n, dtype=np.int32)
        dout = np.zeros((n, 32), dtype=np.uint8)
        self._ck(call(_ptr(base), o.ctypes.data, l.ctypes.data, n, cl.ctypes.data, dg.ctypes.data if dg is not None else None,
                      _ptr(buf) if buf is not None else None, ooff.ctypes.data, status.ctypes.data, dout.ctypes.data))
        good = (status == _lib.DEC_OK) | (status == _lib.DEC_BAD_DIGEST)
        return status, None if buf is None else _split(buf, ooff, cl, good), dout

    # -- f3, read side: archives ---------------------------------------------------------------
    def reader(self, didx: bytes, crypt: "Crypt | None" = None, cache_bytes: int = 0) -> "Reader":
        """Byte ranges of the archive a .didx image describes, served from a cache of verified chunks in device memory
        (pbsgpu_reader_open).  `crypt` decrypts encrypted chunks and checks their keyed digests; `cache_bytes` 0 means
        256 MiB, and the cache always holds at least the largest chunk."""
        return Reader(self, didx, crypt, cache_bytes)

    def reader_fidx(self, fidx: bytes, crypt: "Crypt | None" = None, cache_bytes: int = 0) -> "Reader":
        """The same reader over a disk image's .fidx (pbsgpu_reader_open_fidx): byte ranges of the image; payload reads
        are refused, an image has no pxar headers."""
        return Reader(self, fidx, crypt, cache_bytes, fixed=True)

    # -- f3, encrypt mode -----------------------------------------------------------------------
    def crypt(self, key: bytes) -> "Crypt":
        """Handle for one 32-byte AES-256 key (pbsgpu_crypt_create); close() zeroes its key material."""
        return Crypt(self, key)

    def blob_encode_batch_enc(self, crypt: "Crypt", mode: str, base, off, length, iv: bytes):
        """Encrypted DataBlobs (AES-256-GCM, pbsgpu_blob_encode_batch_enc) of n ranges: the payload is `mode`'s zstd
        frame ("z", "lz", "lze", "lzh", "lzl", "lzc") where smaller, else the raw chunk ("raw": always).  `iv` holds n x 16 bytes, one
        IV per blob; an IV must never be used twice under one key (draw them with os.urandom).
        -> list of n `bytes` blobs, crc[n]."""
        def enc(h, base, o, l, n, *outputs):
            ivs = np.frombuffer(bytes(iv), dtype=np.uint8)
            if len(ivs) != 16 * n:
                raise ValueError("iv must hold 16 bytes per range")
            if mode not in BLOB_MODES or mode is None:
                raise ValueError(f"unknown blob mode {mode!r}")
            return self._L.pbsgpu_blob_encode_batch_enc(h, crypt._h, BLOB_MODES[mode], base, o, l, n, ivs.ctypes.data,
                                                        *outputs)
        return self._blob_encode_sized(enc, base, off, length, 44)

    def blob_header(self, crc: int) -> bytes:
        out = np.zeros(12, dtype=np.uint8)
        self._L.pbsgpu_blob_header(int(crc), out.ctypes.data)
        return out.tobytes()

    # -- f1: dynamic index images ---------------------------------------------------------
    def didx_build(self, chunks: np.ndarray, uuid: bytes = b"\0" * 16, ctime: int = 0) -> bytes:
        """Dynamic-index (.didx) image of chunk records in (stream, offset) order; offsets cumulative."""
        rec = np.ascontiguousarray(chunks, dtype=CHUNK_DTYPE)
        size = int(self._L.pbsgpu_didx_size(len(rec)))
        out = np.zeros(size, dtype=np.uint8)
        u = np.frombuffer(bytes(uuid).ljust(16, b"\0")[:16], dtype=np.uint8)
        self._ck(self._L.pbsgpu_didx_build(self._h, rec.ctypes.data if len(rec) else None, len(rec), u.ctypes.data,
                                           int(ctime), out.ctypes.data, size))
        return out.tobytes()

    def didx_parse(self, image: bytes, verify: bool = True):
        """-> (ends u64[n], digests u8[n,32]); verify recomputes the index checksum on the GPU."""
        a = np.frombuffer(image, dtype=np.uint8)
        n = C.c_uint64()
        self._ck(self._L.pbsgpu_didx_parse(self._h, a.ctypes.data, len(a), None, None, 0, C.byref(n), 0))
        ends = np.zeros(n.value, dtype=np.uint64)
        dig = np.zeros((n.value, 32), dtype=np.uint8)
        self._ck(self._L.pbsgpu_didx_parse(self._h, a.ctypes.data, len(a), ends.ctypes.data, dig.ctypes.data, n.value,
                                           C.byref(n), 1 if verify else 0))
        return ends, dig

    # -- fixed index images (disk images) ------------------------------------------------------
    def fidx_build(self, digests, size: int, chunk_size: int, uuid: bytes = b"\0" * 16, ctime: int = 0) -> bytes:
        """Fixed-index (.fidx) image of an image of `size` bytes in chunks of `chunk_size`: digests (n x 32 bytes, n =
        ceil(size / chunk_size)) in image order; the checksum is computed on the GPU."""
        d = _digests(digests, "each")
        n = d.size // 32
        out = np.zeros(int(self._L.pbsgpu_fidx_size(n)), dtype=np.uint8)
        u = np.frombuffer(bytes(uuid).ljust(16, b"\0")[:16], dtype=np.uint8)
        self._ck(self._L.pbsgpu_fidx_build(self._h, d.ctypes.data if n else None, n, int(size), int(chunk_size), u.ctypes.data,
                                           int(ctime), out.ctypes.data, len(out)))
        return out.tobytes()

    def fidx_parse(self, image: bytes, verify: bool = True):
        """-> (size, chunk_size, digests u8[n, 32]); verify recomputes the index checksum on the GPU."""
        a = np.frombuffer(bytes(image), dtype=np.uint8)
        n, size, cs = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._ck(self._L.pbsgpu_fidx_parse(self._h, a.ctypes.data, len(a), None, None, None, 0, C.byref(n), 0))
        dig = np.zeros((n.value, 32), dtype=np.uint8)
        self._ck(self._L.pbsgpu_fidx_parse(self._h, a.ctypes.data, len(a), C.byref(size), C.byref(cs), dig.ctypes.data,
                                           n.value, C.byref(n), 1 if verify else 0))
        return int(size.value), int(cs.value), dig

    # -- misc ---------------------------------------------------------------------------
    def digest_set(self, capacity_hint: int = 1 << 16) -> "DigestSet":
        return DigestSet(self, capacity_hint)

    def stream(self, cfg: Cfg, digest_set: "DigestSet | None" = None) -> "Stream":
        return Stream(self, cfg, digest_set)

    def host_alloc(self, nbytes: int) -> np.ndarray:
        """Pinned host staging owned by the library (what the Go side would fill)."""
        p = self._L.pbsgpu_host_alloc(self._h, nbytes)
        if not p:
            raise PbsGpuError(_lib.ENOMEM, f"pinned allocation of {nbytes} bytes failed")
        arr = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))
        arr = arr.view(_PinnedArray)
        arr._engine, arr._addr = self, p
        return arr

    def host_free(self, arr):
        addr = getattr(arr, "_addr", None)
        if addr:
            self._L.pbsgpu_host_free(self._h, addr)
            arr._addr = None

    def corpus_fill(self, corpus: Corpus, first_file: int, n_files: int, dst_dev, stride: int):
        self._ck(self._L.pbsgpu_corpus_fill(self._h, C.byref(corpus), first_file, n_files, _ptr(dst_dev), stride))


class _PinnedArray(np.ndarray):
    _engine = None
    _addr = None


class Job:
    """An in-flight batch (pbsgpu_batch_submit); several may overlap on the GPU."""

    def __init__(self, eng: Engine, h, cap: int, keepalive):
        self._eng, self._h, self._cap, self._keep = eng, h, cap, keepalive

    def wait(self):
        out = np.zeros(self._cap, dtype=CHUNK_DTYPE)
        n_out = C.c_uint64()
        t = Timing()
        h = self._h
        rc = self._eng._L.pbsgpu_batch_wait(h, out.ctypes.data, self._cap, C.byref(n_out), C.byref(t))
        if rc == _lib.ERANGE:                       # the job stays valid: retry with the reported capacity
            self._cap = int(n_out.value)
            out = np.zeros(self._cap, dtype=CHUNK_DTYPE)
            rc = self._eng._L.pbsgpu_batch_wait(h, out.ctypes.data, self._cap, C.byref(n_out), C.byref(t))
        self._h = None
        self._eng._ck(rc)
        self._keep = None
        return out[: n_out.value], t.as_dict()

    def wait_input(self):
        """Blocks until the device no longer reads the input buffer (pbsgpu_batch_wait_input); the job stays in flight."""
        self._eng._ck(self._eng._L.pbsgpu_batch_wait_input(self._h))
        self._keep = None

    def input_done(self) -> bool:
        """Non-blocking form of wait_input."""
        rc = self._eng._L.pbsgpu_batch_input_done(self._h)
        if rc < 0:
            self._eng._ck(rc)
        return rc == 1

    def free(self):
        """Abandon the job (pbsgpu_batch_free)."""
        if self._h is not None:
            self._eng._L.pbsgpu_batch_free(self._h)
            self._h, self._keep = None, None


class _Handle:
    """A library object that lives inside an Engine's context: close() calls the C function `_destroy` names once, and
    only while the engine is still open (closing the engine frees everything in its context)."""
    _destroy = ""
    _h = None

    def close(self):
        if self._h and self._eng._h:
            getattr(self._eng._L, self._destroy)(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Crypt(_Handle):
    """One AES-256 key of encrypt mode on the engine's device (pbsgpu_crypt_create / _destroy)."""
    _destroy = "pbsgpu_crypt_destroy"

    def __init__(self, eng: Engine, key: bytes):
        k = np.frombuffer(bytes(key), dtype=np.uint8)
        if len(k) != 32:
            raise ValueError("the key must be 32 bytes")
        self._eng = eng
        h = C.c_void_p()
        eng._ck(eng._L.pbsgpu_crypt_create(eng._h, k.ctypes.data, C.byref(h)))
        self._h = h


def _blob_args(blobs):
    """Reader.read's `blobs` -> (base, blob_off u64[k], blob_len u64[k], blob_chunk u64[k])."""
    if isinstance(blobs, tuple):
        base, bo, bl, bc = blobs
        bo, bl = Engine._offlen(bo, bl)
        bc = np.ascontiguousarray(bc, dtype=np.uint64)
        if bc.shape != bo.shape:
            raise ValueError("blob chunks must hold one index per blob")
        return base, bo, bl, bc
    items = list(blobs.items())
    base, bo, bl = _join([b for _, b in items])
    return base, bo, bl, np.array([c for c, _ in items], dtype=np.uint64)


class Reader(_Handle):
    """An archive reader on the engine's device (pbsgpu_reader_*): plan() names the chunks a read needs that the cache
    lacks, read() verifies the blobs it is given into the cache and copies the ranges out of it."""
    _destroy = "pbsgpu_reader_close"

    def __init__(self, eng: Engine, index: bytes, crypt: "Crypt | None", cache_bytes: int, fixed: bool = False):
        a = np.frombuffer(bytes(index), dtype=np.uint8)
        self._eng, self._crypt = eng, crypt   # the crypt handle must outlive the reader
        h = C.c_void_p()
        op = eng._L.pbsgpu_reader_open_fidx if fixed else eng._L.pbsgpu_reader_open
        eng._ck(op(eng._h, a.ctypes.data, len(a), crypt._h if crypt is not None else None, int(cache_bytes), C.byref(h)))
        self._h = h

    @property
    def size(self) -> int:
        """The archive's length (the index's last end offset)."""
        return int(self._eng._L.pbsgpu_reader_size(self._h))

    def plan(self, off, length, payload: bool = False, sparse: bool = False):
        """The chunks the ranges touch that the cache does not hold -> (chunk indices u64[k] ascending, digests
        u8[k, 32]).  payload: the ranges are (payload offset, file size) of files, their 16-byte headers included.
        sparse (a .fidx reader only): leave out the zero chunks, which read_sparse serves without a blob."""
        o, l = Engine._offlen(off, length)
        flags = (_lib.READ_PAYLOAD if payload else 0) | (_lib.READ_SPARSE if sparse else 0)
        return self._plan(lambda *out: self._eng._L.pbsgpu_reader_plan(self._h, o.ctypes.data, l.ctypes.data, len(o),
                                                                       flags, *out))

    def _plan(self, call):
        """A plan call given its trailing (chunk, digest, cap, n_out) arguments: sized first, then filled."""
        n = C.c_uint64()
        rc = call(None, None, 0, C.byref(n))
        if rc != _lib.ERANGE:
            self._eng._ck(rc)
        chunks = np.zeros(n.value, dtype=np.uint64)
        dig = np.zeros((n.value, 32), dtype=np.uint8)
        if n.value:
            self._eng._ck(call(chunks.ctypes.data, dig.ctypes.data, n.value, C.byref(n)))
        return chunks, dig

    @staticmethod
    def _file_ranges(file_off, file_size, pos, length):
        """File-content ranges -> four u64 arrays of one shape."""
        a = [np.ascontiguousarray(x, dtype=np.uint64).reshape(-1) for x in (file_off, file_size, pos, length)]
        if len({x.shape for x in a}) != 1:
            raise ValueError("file_off, file_size, pos and length must have one entry per range")
        return a

    def plan_file_sparse(self, file_off, file_size, pos, length):
        """The chunks that ranges of file contents need and the cache lacks, leaving out the zero chunks
        (pbsgpu_reader_plan_file_sparse) -> (chunk indices u64[k] ascending, digests u8[k, 32]).  Range i is the content
        bytes [pos[i], pos[i] + length[i]) of the file whose PAYLOAD header is at file_off[i] and whose size is
        file_size[i]; a range at pos 0 also reads that header."""
        fo, fs, p, l = self._file_ranges(file_off, file_size, pos, length)
        return self._plan(lambda *out: self._eng._L.pbsgpu_reader_plan_file_sparse(
            self._h, fo.ctypes.data, fs.ctypes.data, p.ctypes.data, l.ctypes.data, len(fo), *out))

    def read(self, off, length, blobs, payload: bool = False, out: str = "host"):
        """Read ranges (pbsgpu_reader_read).  `blobs`: {chunk index: DataBlob bytes}, or (base, off[k], len[k], chunk[k])
        with a host or device base; their chunks are verified into the cache, then the ranges are copied out of it.
        out: "host" (numpy) or "device" (a torch CUDA tensor).
        -> (status int32[n] (DEC_* values), data, blob_status int32[k]); data holds per range `bytes` ("host") or a
        tensor view ("device"), None where the status is not DEC_OK."""
        if out not in ("host", "device"):
            raise ValueError(f"out must be 'host' or 'device', not {out!r}")
        o, l = Engine._offlen(off, length)
        base, bo, bl, bc = _blob_args(blobs)
        n, k = len(o), len(bo)
        ooff, total = _offsets(l)
        buf = self._eng._alloc(total, out)
        status = np.zeros(n, dtype=np.int32)
        bst = np.zeros(k, dtype=np.int32)
        self._eng._ck(self._eng._L.pbsgpu_reader_read(
            self._h, o.ctypes.data, l.ctypes.data, n, _lib.READ_PAYLOAD if payload else 0, _ptr(base), bo.ctypes.data,
            bl.ctypes.data, bc.ctypes.data, k, _ptr(buf), ooff.ctypes.data, status.ctypes.data, bst.ctypes.data))
        return status, _split(buf, ooff, l, status == _lib.DEC_OK), bst

    def read_deflate(self, off, length, blobs, payload: bool = False, more=None, lzc: bool = False):
        """read() whose outputs are the ranges' raw Deflate streams (pbsgpu_reader_read_deflate): the ranges are
        deflated on the device.  more: per range, a later call continues its stream (length a multiple of
        DEFLATE_SEGMENT).  lzc: the streams of Engine.deflate_batch_lzc instead of deflate_batch.  `blobs` as in
        read().  -> (status int32[n], streams (bytes, None where the status is not DEC_OK), crc32 u32[n],
        blob_status int32[k])"""
        o, l = Engine._offlen(off, length)
        base, bo, bl, bc = _blob_args(blobs)
        n, k = len(o), len(bo)
        ooff, total, m = _deflate_layout(l, more)
        buf = self._eng._alloc(total, "host")
        olen = np.zeros(n, dtype=np.uint64)
        crc = np.zeros(n, dtype=np.uint32)
        status = np.zeros(n, dtype=np.int32)
        bst = np.zeros(k, dtype=np.int32)
        self._eng._ck(self._eng._L.pbsgpu_reader_read_deflate(
            self._h, o.ctypes.data, l.ctypes.data, n,
            (_lib.READ_PAYLOAD if payload else 0) | (_lib.READ_DEFLATE_LZC if lzc else 0), None if m is None else m.ctypes.data, _ptr(base), bo.ctypes.data, bl.ctypes.data, bc.ctypes.data, k,
            buf.ctypes.data, ooff.ctypes.data, olen.ctypes.data, crc.ctypes.data, status.ctypes.data, bst.ctypes.data))
        return status, _split(buf, ooff, olen, status == _lib.DEC_OK), crc, bst


    def read_sparse(self, off, length, blobs):
        """Read ranges of a disk image sparsely (pbsgpu_reader_read_sparse): zero chunks need no blob, and per range
        only the data extents -- the maximal runs of 4 KiB image-aligned block parts that are not all zero -- come
        back.  `blobs` as in read().  -> (status int32[n], per range (extents [(image offset, length)], packed data
        bytes) or None where the status is not DEC_OK, blob_status int32[k])"""
        o, l = Engine._offlen(off, length)
        return self._sparse(o, l, blobs, lambda *a: self._eng._L.pbsgpu_reader_read_sparse(
            self._h, o.ctypes.data, l.ctypes.data, len(o), 0, *a))

    def read_file_sparse(self, file_off, file_size, pos, length, blobs):
        """Read ranges of file contents sparsely (pbsgpu_reader_read_file_sparse): ranges as in plan_file_sparse, zero
        chunks need no blob, and per range only the data extents -- the maximal runs of block parts that are not all
        zero, in 4 KiB blocks aligned to the file's content start -- come back.  A range at pos 0 checks its file's
        PAYLOAD header.  `blobs` as in read().  -> (status int32[n], per range (extents [(content offset, length)],
        packed data bytes) or None where the status is not DEC_OK, blob_status int32[k])"""
        fo, fs, p, l = self._file_ranges(file_off, file_size, pos, length)
        return self._sparse(p, l, blobs, lambda *a: self._eng._L.pbsgpu_reader_read_file_sparse(
            self._h, fo.ctypes.data, fs.ctypes.data, p.ctypes.data, l.ctypes.data, len(fo), *a))

    def _sparse(self, at, length, blobs, call):
        """A sparse read given its block coordinates (at, length) and a call that takes the trailing arguments from
        the blobs on."""
        base, bo, bl, bc = _blob_args(blobs)
        n, k = len(at), len(bo)
        ooff, total = _offsets(length)
        buf = self._eng._alloc(total, "host")
        bs = _lib.SPARSE_BLOCK
        parts = [(int(a) + int(b) - 1) // bs - int(a) // bs + 1 if b else 0 for a, b in zip(at, length)]
        cap = sum((p + 1) // 2 for p in parts)
        ext = np.zeros((max(1, cap), 2), dtype=np.uint64)
        first = np.zeros(n + 1, dtype=np.uint64)
        status = np.zeros(n, dtype=np.int32)
        bst = np.zeros(k, dtype=np.int32)
        self._eng._ck(call(_ptr(base), bo.ctypes.data, bl.ctypes.data, bc.ctypes.data, k, buf.ctypes.data,
                           ooff.ctypes.data, ext.ctypes.data, cap, first.ctypes.data, status.ctypes.data,
                           bst.ctypes.data))
        data = []
        for i in range(n):
            if status[i] != _lib.DEC_OK:
                data.append(None)
                continue
            e = [(int(a), int(b)) for a, b in ext[int(first[i]): int(first[i + 1])]]
            data.append((e, buf[int(ooff[i]): int(ooff[i]) + sum(b for _, b in e)].tobytes()))
        return status, data, bst


class DigestSet(_Handle):
    """Known-digest set on the device (reference: dedup seed, commit.go:286-294, :324-329)."""
    _destroy = "pbsgpu_set_destroy"

    def __init__(self, eng: Engine, capacity_hint: int):
        self._eng = eng
        h = C.c_void_p()
        eng._ck(eng._L.pbsgpu_set_create(eng._h, capacity_hint, C.byref(h)))
        self._h = h

    def __len__(self):
        c = C.c_uint64()
        self._eng._ck(self._eng._L.pbsgpu_set_count(self._h, C.byref(c)))
        return int(c.value)

    def _run(self, fn, digests):
        d = np.ascontiguousarray(digests, dtype=np.uint8).reshape(-1, 32)
        hit = np.zeros(len(d), dtype=np.uint8)
        self._eng._ck(fn(self._h, d.ctypes.data if len(d) else None, len(d), hit.ctypes.data if len(d) else None))
        return hit

    def insert(self, digests) -> np.ndarray:
        """Insert; returns hit[i] = 1 if digest i was already known (before or earlier in this call)."""
        return self._run(self._eng._L.pbsgpu_set_insert, digests)

    def probe(self, digests) -> np.ndarray:
        return self._run(self._eng._L.pbsgpu_set_probe, digests)

    def allgather(self, comm: "NcclComm", digests) -> np.ndarray:
        """The ONE multi-GPU exchange step (pbsgpu_set_allgather): every rank contributes its digests, every replica
        inserts all of them in global (rank, index) order; returns this rank's flags."""
        return self._run(lambda h, *a: self._eng._L.pbsgpu_set_allgather(h, comm._h, *a), digests)

    def _seed(self, fn, image) -> int:
        a = np.frombuffer(bytes(image), dtype=np.uint8)
        n = C.c_uint64()
        self._eng._ck(fn(self._h, a.ctypes.data, len(a), C.byref(n)))
        return int(n.value)

    def seed_didx(self, image: bytes) -> int:
        return self._seed(self._eng._L.pbsgpu_set_seed_didx, image)

    def seed_fidx(self, image: bytes) -> int:
        """Seed from the previous snapshot's .fidx of the same image (pbsgpu_set_seed_fidx); returns its chunk count."""
        return self._seed(self._eng._L.pbsgpu_set_seed_fidx, image)


class NcclComm:
    """An ncclComm_t created through the C ABI's helpers (no torch): rank 0 makes the unique id, every rank passes
    the same 128 bytes (distributed by whatever channel the ranks share) to pbsgpu_nccl_comm_create."""

    def __init__(self, eng: Engine, unique_id: bytes, nranks: int, rank: int):
        self._eng = eng
        ida = np.frombuffer(bytes(unique_id), dtype=np.uint8)
        if len(ida) != 128:
            raise ValueError("NCCL unique id is 128 bytes")
        h = C.c_void_p()
        eng._ck(eng._L.pbsgpu_nccl_comm_create(eng._h, ida.ctypes.data, nranks, rank, C.byref(h)))
        self._h = h

    @staticmethod
    def unique_id() -> bytes:
        out = np.zeros(128, dtype=np.uint8)
        rc = _lib.lib().pbsgpu_nccl_unique_id(out.ctypes.data)
        if rc:
            raise PbsGpuError(rc, "NCCL unavailable (libnccl.so.2 not loadable; set PBSGPU_NCCL_LIB)")
        return out.tobytes()

    def close(self):
        if getattr(self, "_h", None):
            self._eng._L.pbsgpu_nccl_comm_destroy(self._h)
            self._h = None


class Stream(_Handle):
    """Streaming form: one io.Reader-like byte stream, state carried across writes."""
    _destroy = "pbsgpu_stream_close"

    def __init__(self, eng: Engine, cfg: Cfg, digest_set: DigestSet | None):
        self._eng = eng
        self._max = int(cfg.max)
        h = C.c_void_p()
        eng._ck(eng._L.pbsgpu_stream_open(eng._h, C.byref(cfg), digest_set._h if digest_set else None, C.byref(h)))
        self._h = h

    def write(self, data):
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
        self._eng._ck(self._eng._L.pbsgpu_stream_write(self._h, a.ctypes.data if len(a) else None, len(a)))

    def suggest(self, offset: int):
        """Suggested boundary (a file's PAYLOAD header starts here) -- pbsgpu_stream_suggest."""
        self._eng._ck(self._eng._L.pbsgpu_stream_suggest(self._h, int(offset)))

    @property
    def position(self) -> int:
        return int(self._eng._L.pbsgpu_stream_position(self._h))

    def reserve(self) -> np.ndarray:
        """A pinned staging slot owned by the stream; fill a prefix and call commit(n)."""
        p = C.c_void_p()
        self._eng._ck(self._eng._L.pbsgpu_stream_reserve(self._h, C.byref(p)))
        n = int(self._eng._L.pbsgpu_stream_slot_bytes(self._h))
        return np.ctypeslib.as_array((C.c_uint8 * n).from_address(p.value))

    def commit(self, n: int):
        self._eng._ck(self._eng._L.pbsgpu_stream_commit(self._h, int(n)))

    def poll(self, cap: int = 4096) -> np.ndarray:
        out = np.zeros(cap, dtype=CHUNK_DTYPE)
        n = C.c_uint64()
        self._eng._ck(self._eng._L.pbsgpu_stream_poll(self._h, out.ctypes.data, cap, C.byref(n)))
        return out[: n.value]

    def blob_mode(self, mode: str | None):
        """DataBlobs for the new chunks (pbsgpu_stream_blob_mode), set before the first byte: None (no blobs), "raw",
        "z", "lz", "lze", "lzh", "lzl" or "lzc" -- the encoders of Engine.blob_encode_batch, _z, _lz, _lze, _lzh, _lzl
        and _lzc."""
        if mode not in BLOB_MODES:
            raise ValueError(f"blob mode must be one of {list(BLOB_MODES)}, not {mode!r}")
        self._eng._ck(self._eng._L.pbsgpu_stream_blob_mode(self._h, BLOB_MODES[mode]))

    def crypt(self, crypt: "Crypt", iv_seed: bytes | None = None):
        """Encrypt mode (pbsgpu_stream_crypt), set before the first byte: keyed digests, and encrypted blobs whose IVs
        come from the OS CSPRNG -- or, with a 32-byte `iv_seed` (tests), IV_k = SHA-256(iv_seed || k u64 LE)[:16]."""
        seed = None
        if iv_seed is not None:
            seed = np.frombuffer(bytes(iv_seed), dtype=np.uint8)
            if len(seed) != 32:
                raise ValueError("iv_seed must be 32 bytes")
        self._crypt = crypt   # the handle must outlive the stream
        self._eng._ck(self._eng._L.pbsgpu_stream_crypt(self._h, crypt._h, seed.ctypes.data if seed is not None else None))

    def poll_blobs(self, out_cap: int = 0) -> list[bytes]:
        """Every blob available now, in order: blob k belongs to the k-th record without CHUNK_KNOWN."""
        L = self._eng._L
        want = max(int(out_cap), int(L.pbsgpu_blob_size_enc(self._max)), 1 << 24)
        if getattr(self, "_blob_buf", None) is None or len(self._blob_buf) < want:
            self._blob_buf = np.empty(want, dtype=np.uint8)
        out = self._blob_buf
        lens = np.zeros(4096, dtype=np.uint64)
        n = C.c_uint64()
        blobs = []
        while True:
            self._eng._ck(L.pbsgpu_stream_poll_blobs(self._h, out.ctypes.data, len(out), lens.ctypes.data, len(lens), C.byref(n)))
            pos = 0
            for k in range(n.value):
                blobs.append(out[pos: pos + int(lens[k])].tobytes())
                pos += int(lens[k])
            if n.value == 0:
                return blobs

    def hash_range(self, offset: int, length: int):
        """Register [offset, offset + length) for XXH3-64 before its bytes are written (pbsgpu_stream_hash_range)."""
        self._eng._ck(self._eng._L.pbsgpu_stream_hash_range(self._h, int(offset), int(length)))

    def poll_hashes(self, cap: int = 1 << 16) -> np.ndarray:
        """Every XXH3-64 of the registered ranges available now, in registration order (`cap` per C call)."""
        out = np.zeros(cap, dtype=np.uint64)
        n = C.c_uint64()

        def poll():
            self._eng._ck(self._eng._L.pbsgpu_stream_poll_hashes(self._h, out.ctypes.data, cap, C.byref(n)))
            return out[: n.value].copy()
        return self._drain(poll, np.uint64)

    def finish(self) -> np.ndarray:
        self._eng._ck(self._eng._L.pbsgpu_stream_finish(self._h))
        return self._drain(self.poll, CHUNK_DTYPE)

    @staticmethod
    def _drain(poll, dtype) -> np.ndarray:
        """Everything `poll` returns until it returns nothing, concatenated."""
        parts = []
        while len(p := poll()):
            parts.append(p)
        return np.concatenate(parts) if parts else np.zeros(0, dtype=dtype)


def corpus(seed: int, file_len: int, block_len: int = 4 << 20, run_blocks: int = 8, dup_permille: int = 0,
           edit_mode: int = 0, edit_thresh16: int = 655, edit_seed: int = 5) -> Corpus:
    return Corpus(seed, file_len, block_len, run_blocks, dup_permille, edit_mode, edit_thresh16, edit_seed)
