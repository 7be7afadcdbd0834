"""Mirror of the reference's dedup split-archive writer surface, for the hot path only.

Reference (Go, module github.com/pbs-plus/pxar/transfer, call sites in
internal/pxarmount/commit.go):
    writer, err := transfer.NewRemoteDedupSplitArchiveWriter(ctx, session, meta, payload, origPayloadIdx)   :329
    err = writer.WriteEntryReader(entry, reader, size)                                                      :720, :858
    err = writer.Finish()                                                                                   :383
Inside WriteEntryReader the module pulls the reader's bytes, runs the buzhash scan,
cuts, SHA-256s every chunk, asks the session whether the digest is known and uploads
only new chunks.  This mirror keeps the names and the pull-from-a-reader contract but
batches the files: entries are queued and pushed through the GPU engine in one batch on
Flush()/Finish() (SURVEY.md section 8f item 2).  `upload` is a callback (the HTTP/2 upload is out of scope).

One reader: PayloadReader -- the mirror of SplitArchiveReader.PayloadReaderAt() (pxarfs.go:38, :409-412): byte ranges
and whole files of a payload stream, served through pbsgpu_reader_* from a cache of verified chunks on the GPU; the
chunk files come from a `chunk_source` callback (reading the datastore is out of scope).

Two writers:
  * PayloadStreamWriter -- the LAYOUT-FAITHFUL one and the default for a drop-in: it produces the pxar v2 payload
    stream the production chunker sees (PAYLOAD_START marker, then per file a 16-byte PAYLOAD header + content,
    concatenated: internal/pxarmount/pxarfs.go:408-411), chunks THAT stream through pbsgpu_stream_* with a suggested
    boundary at every file start, returns each entry's payload offset (what the mpxar PAYLOAD_REF stores) and
    supports WriteEntryRef (chunk reuse from the previous .ppxar.didx, commit.go:752, :848-860).
  * DedupWriter -- per-file batching (every file its own stream).  Faster for many small files, but its index does NOT
    describe a ppxar payload stream: use it for dedup statistics / digest computation, not to write .ppxar.didx.

And for disk images (`.img.fidx` archives): FixedIndexWriter -- fixed-size chunks through the batch call, fed in slices;
restore_image -- the sparse restore: zero chunks are served by digest and only the data extents are written.
PayloadReader.RestoreFiles -- the same for the files of a payload stream, restored into a directory.

Restore as zip (reference internal/pxar/zip.go): ZipWriter -- files of a PayloadReader deflated on the GPU
(pbsgpu_reader_read_deflate) inside a zip container written by pbsgpu_zip_*.
"""
from __future__ import annotations

import io
import os
import stat
import zlib
from collections import deque
from dataclasses import dataclass, field
from typing import BinaryIO, Callable

import numpy as np

from . import _lib
from ._lib import CHUNK_DTYPE, CHUNK_KNOWN, Cfg
from . import engine as _engine
from .engine import DigestSet, Engine


@dataclass
class Entry:
    """The two fields of pxar.Entry the hot path reads (commit.go:710-715)."""
    Path: str
    FileSize: int


@dataclass
class IndexRecord:
    """One dynamic-index entry the writer appends per chunk: (end offset, digest)."""
    path: str
    end_off: int
    digest: bytes
    known: bool


@dataclass
class DedupWriter:
    engine: Engine
    config: Cfg
    known: DigestSet | None = None
    upload: Callable[[bytes, bytes], None] | None = None   # (digest, chunk bytes) for NEW chunks
    # (digest, DataBlob) for NEW chunks: the body of POST /dynamic_chunk (log_cleanup.go:19-31), rendered for all new
    # chunks of a flush by ONE pbsgpu_blob_encode_batch_z call (zstd frame where smaller, CRC-32 from the GPU)
    upload_blob: Callable[[bytes, bytes], None] | None = None
    batch_bytes: int = 1 << 30
    # "z": frames of RLE and raw blocks; "lz": also compressed blocks from the LZ77 match stage (pbsgpu_blob_encode_batch_lz);
    # "lze": those blocks also through zstd's entropy stage (pbsgpu_blob_encode_batch_lze); "lzh": with Huffman literals
    # whatever their largest value, for binary data (pbsgpu_blob_encode_batch_lzh); "lzl": also long matches anywhere
    # earlier in the chunk, for repeats beyond one 128 KiB block (pbsgpu_blob_encode_batch_lzl); "lzc": _lzh with a
    # hash-chain match search over the whole chunk and a lazy parse, for smaller text-like blobs (pbsgpu_blob_encode_batch_lzc)
    blob_compression: str = "z"
    # encrypt mode (CryptMode encrypt, commit.go:314): the 32-byte client key.  Digests become keyed (SHA-256(chunk ||
    # id_key)) and upload_blob receives encrypted blobs (pbsgpu_blob_encode_batch_enc, IVs from os.urandom)
    crypt_key: bytes | None = None
    index: list[IndexRecord] = field(default_factory=list)
    # relPath -> XXH3-64 of the file as uploaded: commitWalkState.backedHashes (commit.go:187, :725), computed on the
    # GPU from the same staged bytes instead of through an io.TeeReader on the host
    backed_hashes: dict[str, int] = field(default_factory=dict)
    _pending: list[tuple[Entry, np.ndarray]] = field(default_factory=list)
    _pending_bytes: int = 0
    _finished: bool = False
    _crypt: object = None

    def __post_init__(self):
        _check_blob_compression(self.blob_compression)
        if self.crypt_key is not None:
            self._crypt = self.engine.crypt(self.crypt_key)

    def WriteEntryReader(self, entry: Entry, reader: BinaryIO, size: int) -> None:
        """Pulls exactly `size` bytes from `reader` (error if it yields fewer, like io.ReadFull)."""
        if self._finished:
            raise RuntimeError("transfer: writer already finished")
        data = reader.read(size) if size else b""
        if len(data) != size:
            raise IOError(f"transfer: short read for {entry.Path}: got {len(data)} of {size} bytes (unexpected EOF)")
        self._pending.append((entry, np.frombuffer(data, dtype=np.uint8)))
        self._pending_bytes += size
        if self._pending_bytes >= self.batch_bytes:
            self.Flush()

    def WriteEntry(self, entry: Entry, data: bytes) -> None:
        self.WriteEntryReader(entry, io.BytesIO(data), len(data))

    def Flush(self) -> None:
        if not self._pending:
            return
        entries, arrs = zip(*self._pending)
        buf, offs, lens = _engine._pack(arrs)
        keyed = {"crypt": self._crypt} if self._crypt is not None else {}
        rec, hashes = self.engine.chunk_digest_batch_xxh3(self.config, buf, offs, lens, self.known, **keyed)
        for e, h in zip(entries, hashes):
            self.backed_hashes[e.Path] = int(h)
        new_chunks = []                                   # (digest, stream, start, end) of the chunks the server lacks
        starts: dict[int, int] = {}
        for r in rec:
            i = int(r["stream"])
            known = bool(r["flags"] & CHUNK_KNOWN)
            s0, e0 = starts.get(i, 0), int(r["end_off"])
            starts[i] = e0
            self.index.append(IndexRecord(entries[i].Path, e0, bytes(r["digest"]), known))
            if not known:
                new_chunks.append((bytes(r["digest"]), i, s0, e0))
        if self.upload is not None:
            for d, i, s0, e0 in new_chunks:
                self.upload(d, arrs[i][s0:e0].tobytes())
        if self.upload_blob is not None and new_chunks:
            boff = np.array([int(offs[i]) + s0 for _, i, s0, _ in new_chunks], dtype=np.uint64)
            blen = np.array([e0 - s0 for _, _, s0, e0 in new_chunks], dtype=np.uint64)
            blobs = _encode_new(self.engine, self._crypt, self.blob_compression, buf, boff, blen)
            for (d, _i, _s, _e), blob in zip(new_chunks, blobs):
                self.upload_blob(d, blob)
        self._pending, self._pending_bytes = [], 0

    def Finish(self) -> list[IndexRecord]:
        self.Flush()
        self._finished = True
        return self.index


def _check_blob_compression(c: str) -> None:
    names = [m for m in _lib.BLOB_MODES if m not in (None, "raw")]
    if c not in names:
        raise ValueError(f"transfer: blob_compression must be {', '.join(map(repr, names[:-1]))} or {names[-1]!r}, "
                         f"not {c!r}")


def _encode_new(engine: Engine, crypt, mode: str, base, off, length) -> list[bytes]:
    """The DataBlobs of new chunks: encrypted with `crypt` under fresh random IVs, else plain by `mode`'s encoder."""
    if crypt is not None:
        blobs, _crc = engine.blob_encode_batch_enc(crypt, mode, base, off, length, os.urandom(16 * len(off)))
    else:
        blobs, _crc = getattr(engine, "blob_encode_batch_" + mode)(base, off, length)
    return blobs


# pxar v2 format constants (upstream pxar crate format/mod.rs; restated, UNVERIFIED against the Go module)
PXAR_PAYLOAD = 0x28147A1B0B7C1A25
PXAR_PAYLOAD_START_MARKER = 0x834C68C2194A4ED2
PXAR_PAYLOAD_TAIL_MARKER = 0x6C72B78B984C81B5


def payload_header(content_len: int) -> bytes:
    """16-byte PAYLOAD header: htype u64 LE, full_size u64 LE (header included) -- pxarfs.go:408-411 skips these 16."""
    return PXAR_PAYLOAD.to_bytes(8, "little") + (16 + content_len).to_bytes(8, "little")


class NotStrictlyGreater(IOError):
    """WriteEntryRef out of order; the message carries the substring the reference matches (commit.go:849)."""


@dataclass
class PayloadStreamWriter:
    """Writes ONE pxar v2 payload stream through the streaming C ABI (see the module docstring)."""
    engine: Engine
    config: Cfg
    known: DigestSet | None = None
    prev_index: tuple[np.ndarray, np.ndarray] | None = None   # (ends u64[], digests u8[n,32]) of the previous .ppxar.didx
    suggest: bool = True             # suggested boundary at every file start (upstream PayloadChunker); False = plain chunker
    index: list[tuple[int, bytes, bool]] = field(default_factory=list)   # (end offset in the NEW stream, digest, known)
    payload_offsets: dict[str, int] = field(default_factory=dict)        # entry path -> offset of its PAYLOAD header
    # (digest, DataBlob) for NEW chunks, encoded on the GPU from the stream's windows (pbsgpu_stream_blob_mode) with the
    # encoder `blob_compression` names ("z", "lz", "lze", "lzh", "lzl" or "lzc", as for DedupWriter).  Chunks injected by WriteEntryRef get none.
    upload_blob: Callable[[bytes, bytes], None] | None = None
    blob_compression: str = "z"
    # hash_files: relPath -> XXH3-64 of every file written through WriteEntryReader in backed_hashes
    # (commitWalkState.backedHashes, commit.go:725), hashed on the GPU from the stream's windows
    # (pbsgpu_stream_hash_range).  Off by default: a stream with no hash ranges does no hashing work.
    hash_files: bool = False
    backed_hashes: dict[str, int] = field(default_factory=dict)
    # encrypt mode: the 32-byte client key (as DedupWriter.crypt_key); the stream draws the blobs' IVs from the OS CSPRNG
    crypt_key: bytes | None = None
    _crypt: object = None
    _stream: object = None
    _seg_base: int = 0               # offset in the new stream at which the current pbsgpu stream starts
    _last_ref: int = -1
    _finished: bool = False
    _new: list = field(default_factory=list)          # digests of new records still waiting for their blob
    _blobs: list = field(default_factory=list)        # blobs still waiting for their record
    _hashed: deque = field(default_factory=deque)     # paths whose hash the stream has not returned yet

    def __post_init__(self):
        _check_blob_compression(self.blob_compression)
        if self.crypt_key is not None:
            self._crypt = self.engine.crypt(self.crypt_key)
        self._open()
        self._raw(PXAR_PAYLOAD_START_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little"))

    # -- plumbing ---------------------------------------------------------------------------------------------
    def _open(self):
        self._stream = self.engine.stream(self.config, self.known)
        if self._crypt is not None:
            self._stream.crypt(self._crypt)
        if self.upload_blob is not None:
            self._stream.blob_mode(self.blob_compression)

    def _raw(self, data: bytes):
        self._stream.write(np.frombuffer(data, dtype=np.uint8))

    @property
    def position(self) -> int:
        return self._seg_base + self._stream.position

    def _drain(self, final: bool):
        rec = self._stream.finish() if final else self._stream.poll(1 << 16)
        for r in rec:
            known = bool(r["flags"] & CHUNK_KNOWN)
            self.index.append((self._seg_base + int(r["end_off"]), bytes(r["digest"]), known))
            if self.upload_blob is not None and not known:
                self._new.append(bytes(r["digest"]))
        if self.upload_blob is not None:
            # blob k belongs to the k-th new record; either side may run ahead of the other between polls
            self._blobs += self._stream.poll_blobs()
            k = min(len(self._new), len(self._blobs))
            for d, b in zip(self._new[:k], self._blobs[:k]):
                self.upload_blob(d, b)
            del self._new[:k], self._blobs[:k]
        if self._hashed:
            for h in self._stream.poll_hashes():
                self.backed_hashes[self._hashed.popleft()] = int(h)
        if final and (self._new or self._blobs or self._hashed):
            raise RuntimeError("transfer: the stream finished with blobs or hashes unaccounted for")

    # -- ArchiveWriter surface (commit.go:183) -------------------------------------------------------------------
    def WriteEntryReader(self, entry: Entry, reader: BinaryIO, size: int) -> int:
        """commit.go:720, :858.  Returns the entry's payload offset."""
        if self._finished:
            raise RuntimeError("transfer: writer already finished")
        off = self.position
        if self.suggest and self._stream.position > 0:
            self._stream.suggest(self._stream.position)
        if self.hash_files:
            self._stream.hash_range(self._stream.position + 16, size)
            self._hashed.append(entry.Path)
        self._raw(payload_header(size))
        left = size
        while left:
            slot = self._stream.reserve()
            want = min(left, len(slot))
            data = reader.read(want)
            if not data:
                self._stream.commit(0)
                raise IOError(f"transfer: short read for {entry.Path}: got {size - left} of {size} bytes (unexpected EOF)")
            slot[: len(data)] = np.frombuffer(data, dtype=np.uint8)
            self._stream.commit(len(data))
            left -= len(data)
        self.payload_offsets[entry.Path] = off
        self._drain(False)
        return off

    def WriteEntryRef(self, entry: Entry, payload_offset: int) -> int:
        """commit.go:752, :848: reuse the previous snapshot's chunks that hold [payload_offset, +16+FileSize) without
        reading the content.  The running chunk is closed, the old chunks are appended to the new index (their bytes
        become part of the new stream, padding included, as in upstream's chunk injection) and the entry's new payload
        offset is returned.  Offsets must ascend; otherwise the error text contains "not strictly greater" and the
        caller re-encodes through WriteEntryReader (commit.go:849-860)."""
        if self.prev_index is None:
            raise IOError("transfer: WriteEntryRef without a previous payload index")
        if payload_offset <= self._last_ref:
            raise NotStrictlyGreater(f"transfer: payload offset {payload_offset} not strictly greater than previous {self._last_ref}")
        ends, digs = self.prev_index
        lo = int(np.searchsorted(ends, payload_offset, side="right"))
        hi = int(np.searchsorted(ends, payload_offset + 16 + entry.FileSize, side="left"))
        if hi >= len(ends):
            raise IOError(f"transfer: payload range of {entry.Path} lies outside the previous index")
        # close the running chunk: the injected chunks start on a chunk boundary of the new stream
        self._drain(True)
        self._seg_base += self._stream.position
        self._stream.close()
        first_start = int(ends[lo - 1]) if lo else 0
        pos = self._seg_base
        for k in range(lo, hi + 1):
            start = int(ends[k - 1]) if k else 0
            pos += int(ends[k]) - start
            self.index.append((pos, bytes(digs[k]), True))
        new_off = self._seg_base + (payload_offset - first_start)
        self._seg_base = pos
        self._last_ref = payload_offset
        self.payload_offsets[entry.Path] = new_off
        self._open()
        return new_off

    def Finish(self) -> list[tuple[int, bytes, bool]]:
        """commit.go:383: tail marker, final short chunk, index complete."""
        if not self._finished:
            try:
                self._raw(PXAR_PAYLOAD_TAIL_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little"))
                self._drain(True)
            finally:
                self._stream.close()
                self._finished = True
        return self.index

    def didx(self, uuid: bytes = b"\0" * 16, ctime: int = 0) -> bytes:
        """The new .ppxar.didx image (csum on the GPU)."""
        rec = np.zeros(len(self.index), dtype=CHUNK_DTYPE)
        for i, (end, dig, known) in enumerate(self.index):
            rec[i]["end_off"] = end
            rec[i]["digest"] = np.frombuffer(dig, dtype=np.uint8)
            rec[i]["flags"] = CHUNK_KNOWN if known else 0
        return self.engine.didx_build(rec, uuid, ctime)


@dataclass
class FixedIndexWriter:
    """Backs up a disk image as a fixed index (`<name>.img.fidx`): the image is cut at every multiple of `chunk_size`
    (upstream writes 4 MiB chunks), and each chunk is digested on the GPU, probed against `known` (seed it from the
    previous snapshot's index with DigestSet.seed_fidx) and, when new, handed to `upload_blob(digest, blob)` as a
    DataBlob made by the encoder `blob_compression` names ("z", "lz", "lze", "lzh", "lzl" or "lzc", as for DedupWriter).  No
    state crosses a chunk boundary, so the image is fed in slices of any size that are multiples of `chunk_size` -- only
    the last may end inside a chunk -- one batch call per slice, from host memory or straight from device memory."""
    engine: Engine
    chunk_size: int = 4 << 20
    known: DigestSet | None = None
    upload_blob: Callable[[bytes, bytes], None] | None = None
    blob_compression: str = "z"
    # encrypt mode: the 32-byte client key (as DedupWriter.crypt_key): keyed digests and encrypted blobs
    crypt_key: bytes | None = None
    digests: list[bytes] = field(default_factory=list)   # per chunk, in image order
    known_flags: list[bool] = field(default_factory=list)
    size: int = 0                                        # image bytes written so far
    _crypt: object = None
    _ended: bool = False                                 # a slice ended inside a chunk: it was the last

    def __post_init__(self):
        _check_blob_compression(self.blob_compression)
        cs = int(self.chunk_size)
        if cs < 4096 or cs > 16 << 20 or cs & (cs - 1):
            raise ValueError(f"transfer: chunk_size must be a power of two from 4 KiB to 16 MiB, not {cs}")
        if self.crypt_key is not None:
            self._crypt = self.engine.crypt(self.crypt_key)

    def WriteSlice(self, data) -> None:
        """The next bytes of the image: a numpy array or bytes on the host, or a 1-D torch CUDA tensor of uint8."""
        if isinstance(data, (bytes, bytearray, memoryview)):
            data = np.frombuffer(data, dtype=np.uint8)
        n = int(data.numel()) if hasattr(data, "numel") else len(data)
        if n == 0:
            return
        if self._ended:
            raise ValueError("transfer: the image's last slice ended inside a chunk; no slice may follow it")
        cs = int(self.chunk_size)
        rec = self.engine.chunk_digest_batch(None, data, [0], [n], self.known, crypt=self._crypt, fixed_size=cs)
        new = []
        for k, r in enumerate(rec):
            known = bool(r["flags"] & CHUNK_KNOWN)
            self.digests.append(bytes(r["digest"]))
            self.known_flags.append(known)
            if not known:
                new.append(k)
        if self.upload_blob is not None and new:
            boff = np.array(new, dtype=np.uint64) * np.uint64(cs)
            blen = np.minimum(np.uint64(n) - boff, np.uint64(cs))
            for k, blob in zip(new, _encode_new(self.engine, self._crypt, self.blob_compression, data, boff, blen)):
                self.upload_blob(bytes(rec[k]["digest"]), blob)
        self.size += n
        self._ended = n % cs != 0

    def WriteFrom(self, reader: BinaryIO, size: int, slice_bytes: int = 1 << 30) -> None:
        """Pulls exactly `size` bytes from `reader` (io.ReadFull semantics) in slices of `slice_bytes` (rounded down to
        whole chunks)."""
        step = max(int(self.chunk_size), slice_bytes - slice_bytes % int(self.chunk_size))
        left = size
        while left:
            want = min(left, step)
            data = reader.read(want)
            if len(data) != want:
                raise IOError(f"transfer: short read of the image: got {size - left + len(data)} of {size} bytes (unexpected EOF)")
            self.WriteSlice(data)
            left -= want

    def fidx(self, uuid: bytes = b"\0" * 16, ctime: int = 0) -> bytes:
        """The image's .fidx (checksum on the GPU)."""
        return self.engine.fidx_build(b"".join(self.digests), self.size, int(self.chunk_size), uuid, ctime)


_DEC_NAMES = {getattr(_lib, k): k for k in dir(_lib) if k.startswith("DEC_")}


class PayloadReader:
    """Reads a payload stream (.ppxar.didx) the way SplitArchiveReader.PayloadReaderAt() serves PxarFS.readFileContent
    (pxarfs.go:409-412) and restore (format.go:113-132).  Every chunk is decoded and verified on the GPU once (CRC, GCM
    tag with `crypt_key`, zstd, digest against the index) into a device cache of `cache_bytes` (0 = 256 MiB, pxar-mount's
    --cache-size default); reads are copied out of that cache.  `chunk_source(digest)` returns the DataBlob of a chunk
    (the bytes of .chunks/<hex>).  Errors raise IOError naming the first bad range and its status."""

    def __init__(self, engine: Engine, ppxar_didx: bytes, chunk_source: Callable[[bytes], bytes],
                 crypt_key: bytes | None = None, cache_bytes: int = 0):
        self._crypt = engine.crypt(crypt_key) if crypt_key is not None else None
        self._reader = engine.reader(ppxar_didx, self._crypt, cache_bytes)
        self._source = chunk_source

    @property
    def Size(self) -> int:
        return self._reader.size

    def _fetch(self, off: list[int], size: list[int], payload: bool) -> dict[int, bytes]:
        """One plan, one fetch of the missing blobs by digest."""
        chunks, digests = self._reader.plan(off, size, payload)
        return {int(c): self._source(bytes(d)) for c, d in zip(chunks, digests)}

    @staticmethod
    def _check(status, off: list[int], size: list[int], payload: bool) -> None:
        bad = np.flatnonzero(status != _lib.DEC_OK)
        if len(bad):
            i = int(bad[0])
            what = "file at payload offset" if payload else "range at"
            raise IOError(f"transfer: {what} {off[i]} ({size[i]} bytes): {_DEC_NAMES.get(int(status[i]), int(status[i]))}")

    def _read(self, off: list[int], size: list[int], payload: bool) -> list[bytes]:
        """One plan, one fetch, one read."""
        status, data, _ = self._reader.read(off, size, self._fetch(off, size, payload), payload)
        self._check(status, off, size, payload)
        return data

    def _read_deflate(self, off: list[int], size: list[int], payload: bool, more=None, lzc: bool = False):
        """_read whose outputs are raw Deflate streams (with lzc, Engine.deflate_batch_lzc's) -> (streams, crc32s)."""
        status, streams, crc, _ = self._reader.read_deflate(off, size, self._fetch(off, size, payload), payload, more,
                                                            lzc)
        self._check(status, off, size, payload)
        return streams, [int(c) for c in crc]

    def ReadAt(self, off: int, size: int) -> bytes:
        """io.ReaderAt: up to `size` bytes at archive offset `off`; short (possibly empty) at the archive's end."""
        if off < 0 or size < 0:
            raise ValueError("transfer: negative offset or size")
        size = max(0, min(size, self.Size - off))
        return self._read([off], [size], False)[0] if size else b""

    def ReadFileContents(self, files: list[tuple[int, int]]) -> list[bytes]:
        """The contents of files given as (payload offset, size), each checked against its 16-byte PAYLOAD header."""
        if not files:
            return []
        off, size = zip(*files)
        return self._read(list(off), list(size), True)

    def RestoreFiles(self, root: str, entries: list, no_attr: bool = False, slice_bytes: int = 1 << 30) -> None:
        """Restores entries into the directory `root` (reference restoreNormal / restoreFile / restoreSymlink,
        internal/pxar/restore.go): DirEntry, FileEntry and SymlinkEntry items, paths relative to root, a directory
        before what it holds.  File contents are read sparsely (pbsgpu_reader_read_file_sparse): zero chunks are never
        fetched or decoded, and only the data extents come back.  Each file is opened with O_CREAT | O_TRUNC, gets one
        os.pwrite per extent and an os.ftruncate to its size, so its all-zero 4 KiB blocks stay holes.  Files up to
        `slice_bytes` go in batches of about `slice_bytes` file bytes, one plan / fetch / read per batch; a larger file
        is read in pieces of `slice_bytes` (rounded down to a multiple of 4096).  A file whose type and size match the
        entry, and its mtime too unless `no_attr`, is not rewritten (shouldUpdateFile).  Unless `no_attr`, files and
        directories get the entry's permission bits and mtime (owners, xattrs, ACLs and fcaps are not restored).
        Raises IOError naming the first file that cannot be read and its status."""
        piece = max(_lib.SPARSE_BLOCK, int(slice_bytes) // _lib.SPARSE_BLOCK * _lib.SPARSE_BLOCK)
        os.makedirs(root, exist_ok=True)
        dirs, batch, acc = [], [], 0
        for e in entries:
            path = _restore_path(root, e.path)
            if isinstance(e, DirEntry):
                os.makedirs(path, exist_ok=True)
                dirs.append((path, e))
            elif isinstance(e, SymlinkEntry):
                _restore_symlink(path, e.target)
            elif not _should_update(path, e, no_attr):
                if not no_attr:
                    _apply_attrs(path, e)
            elif e.size > piece:
                self._restore_large(path, e, piece, no_attr)
            else:
                if batch and acc + e.size > piece:
                    self._restore_batch(batch, no_attr)
                    batch, acc = [], 0
                batch.append((path, e))
                acc += e.size
        self._restore_batch(batch, no_attr)
        if not no_attr:   # after their contents, deepest first, so writing a file does not move a directory's mtime
            for path, e in reversed(dirs):
                _apply_attrs(path, e)

    def _read_file_sparse(self, what: list[tuple[str, "FileEntry"]], pos: list[int], n: list[int]):
        """One plan, one fetch and one pbsgpu_reader_read_file_sparse of ranges of files -> per range (extents, packed)."""
        fo, fs = [e.payload_offset for _, e in what], [e.size for _, e in what]
        chunks, digests = self._reader.plan_file_sparse(fo, fs, pos, n)
        blobs = {int(c): self._source(bytes(d)) for c, d in zip(chunks, digests)}
        status, data, _ = self._reader.read_file_sparse(fo, fs, pos, n, blobs)
        for (path, e), s in zip(what, status):
            if s != _lib.DEC_OK:
                raise IOError(f"transfer: restore of {path} (payload offset {e.payload_offset}, {e.size} bytes): "
                              f"{_DEC_NAMES.get(int(s), int(s))}")
        return data

    def _restore_batch(self, batch, no_attr: bool) -> None:
        if not batch:
            return
        data = self._read_file_sparse(batch, [0] * len(batch), [e.size for _, e in batch])
        for (path, e), (extents, packed) in zip(batch, data):
            fd = os.open(path, os.O_CREAT | os.O_TRUNC | os.O_WRONLY, 0o666)
            try:
                _write_extents(fd, extents, packed)
                os.ftruncate(fd, e.size)
            finally:
                os.close(fd)
            if not no_attr:
                _apply_attrs(path, e)

    def _restore_large(self, path: str, e: "FileEntry", piece: int, no_attr: bool) -> None:
        fd = os.open(path, os.O_CREAT | os.O_TRUNC | os.O_WRONLY, 0o666)
        try:
            for lo in range(0, e.size, piece):
                (extents, packed), = self._read_file_sparse([(path, e)], [lo], [min(piece, e.size - lo)])
                _write_extents(fd, extents, packed)
            os.ftruncate(fd, e.size)
        finally:
            os.close(fd)
        if not no_attr:
            _apply_attrs(path, e)

    def Close(self) -> None:
        self._reader.close()
        if self._crypt is not None:
            self._crypt.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.Close()


@dataclass
class DirEntry:
    """A directory of PayloadReader.RestoreFiles: path relative to the root, st_mode, mtime in seconds."""
    path: str
    mode: int
    mtime: int


@dataclass
class FileEntry:
    """A regular file of PayloadReader.RestoreFiles: path, st_mode, mtime in seconds, the payload offset of its
    PAYLOAD header (what the mpxar PAYLOAD_REF stores) and its size."""
    path: str
    mode: int
    mtime: int
    payload_offset: int
    size: int


@dataclass
class SymlinkEntry:
    """A symlink of PayloadReader.RestoreFiles: path and target."""
    path: str
    target: str


def _restore_path(root: str, rel: str) -> str:
    """root/rel, refusing a path that leaves root."""
    parts = rel.replace(os.sep, "/").split("/")
    if os.path.isabs(rel) or ".." in parts:
        raise ValueError(f"transfer: restore path {rel!r} leaves the target directory")
    return os.path.join(root, rel)


def _should_update(path: str, e: FileEntry, no_attr: bool) -> bool:
    """The reference's shouldUpdateFile (internal/pxar/restore.go) for a regular file: rewrite it unless a regular file of the
    entry's size, and (unless no_attr) its mtime in seconds, is already there."""
    try:
        st = os.lstat(path)
    except FileNotFoundError:
        return True
    if stat.S_ISDIR(st.st_mode) or stat.S_ISLNK(st.st_mode) or st.st_size != e.size:
        return True
    return not no_attr and int(st.st_mtime) != int(e.mtime)


def _restore_symlink(path: str, target: str) -> None:
    """restoreSymlink: keep a symlink that already points at target, replace one that points elsewhere."""
    try:
        if os.readlink(path) == target:
            return
        os.remove(path)
    except OSError:
        pass
    os.symlink(target, path)


def _apply_attrs(path: str, e) -> None:
    """applyMeta's permission bits and mtime (atime = mtime)."""
    os.chmod(path, e.mode & 0o777)
    os.utime(path, (e.mtime, e.mtime))


def _write_extents(fd: int, extents, packed: bytes) -> None:
    """One os.pwrite per (offset, length) extent of the packed bytes."""
    view, at = memoryview(packed), 0
    for eo, el in extents:
        done = 0
        while done < el:
            done += os.pwrite(fd, view[at + done: at + el], eo + done)
        at += el


def restore_image(engine: Engine, fidx: bytes, chunk_source: Callable[[bytes], bytes], fd: int,
                  crypt_key: bytes | None = None, slice_bytes: int = 1 << 30, cache_bytes: int = 0) -> None:
    """Restores the disk image a `.img.fidx` describes into the file descriptor `fd`, sparsely: per slice of
    `slice_bytes`, one plan that leaves out the zero chunks, one fetch of the named blobs by digest through
    `chunk_source`, one pbsgpu_reader_read_sparse, and an os.pwrite of each data extent; then os.ftruncate to the image's
    size.  Zero chunks are never fetched or decoded, and no all-zero 4 KiB block is written, so the target must read as
    zeros where nothing is written: a new file (which stays thin), or a device the caller zeroed, as upstream's
    skip-zero restore.  `crypt_key` and `cache_bytes` as for PayloadReader.  Raises IOError naming the first chunk whose
    blob fails a check."""
    crypt = engine.crypt(crypt_key) if crypt_key is not None else None
    try:
        reader = engine.reader_fidx(fidx, crypt, cache_bytes)
        try:
            size, step = reader.size, max(1, int(slice_bytes))
            for off in range(0, size, step):
                n = min(step, size - off)
                chunks, digests = reader.plan([off], [n], sparse=True)
                blobs = {int(c): chunk_source(bytes(d)) for c, d in zip(chunks, digests)}
                status, data, bst = reader.read_sparse([off], [n], blobs)
                if status[0] != _lib.DEC_OK:
                    bad = [f"chunk {int(c)} ({bytes(d).hex()})" for c, d, s in zip(chunks, digests, bst) if s != _lib.DEC_OK]
                    where = bad[0] if bad else f"the slice at {off}"
                    raise IOError(f"transfer: image {where}: {_DEC_NAMES.get(int(status[0]), int(status[0]))}")
                _write_extents(fd, *data[0])
            os.ftruncate(fd, size)
        finally:
            reader.close()
    finally:
        if crypt is not None:
            crypt.close()


class ZipWriter:
    """One `<name>.zip` of a restore (reference createZipForSource, internal/pxar/zip.go), written to `w`: directories,
    symlinks (stored, the target as content) and files deflated on the GPU from a PayloadReader.  Every entry but a
    directory has flag bit 3 and a data descriptor; Close writes the central directory.

    AddFiles takes (path, st_mode, mtime, payload offset, size) tuples.  Files up to `piece_bytes` go in batches of
    about `piece_bytes` file bytes, one plan / fetch / read_deflate per batch; a larger file goes in 128 KiB-aligned
    pieces of plain ranges continued with `more`, after one plain read of its 16-byte PAYLOAD header, and its CRC-32 is
    combined from the pieces'.  lzc: deflate with the hash-chain parse (Engine.deflate_batch_lzc), for a smaller zip
    at a lower rate; the default writes the greedy parse's streams."""

    def __init__(self, reader: PayloadReader, w: BinaryIO, piece_bytes: int = 1 << 30, lzc: bool = False):
        self._r, self._w, self._lzc = reader, w, lzc
        self._piece = max(_lib.DEFLATE_SEGMENT, piece_bytes // _lib.DEFLATE_SEGMENT * _lib.DEFLATE_SEGMENT)
        self._pos, self._entries = 0, []

    def _write(self, b: bytes) -> None:
        self._w.write(b)
        self._pos += len(b)

    def _entry(self, name: str, mode: int, mtime: int, method: int, body, crc: int, csize: int, size: int) -> None:
        e = _engine.zip_entry(name.encode(), mode, int(mtime), method, crc, csize, size, self._pos)
        self._write(_engine.zip_local_header(e))
        for part in body:
            self._write(part)
        self._write(_engine.zip_data_descriptor(e))
        self._entries.append(e)

    def AddDirectory(self, path: str, mode: int, mtime: int) -> None:
        name = path if path.endswith("/") else path + "/"
        self._entry(name, mode, mtime, 0, [], 0, 0, 0)

    def AddSymlink(self, path: str, target: str, mode: int, mtime: int) -> None:
        t = target.encode()
        self._entry(path, mode, mtime, 0, [t], zlib.crc32(t), len(t), len(t))

    def AddFiles(self, files: list[tuple[str, int, int, int, int]]) -> None:
        batch, acc = [], 0
        for f in files:
            if f[4] > self._piece:
                self._flush(batch)
                batch, acc = [], 0
                self._large(*f)
                continue
            if batch and acc + f[4] > self._piece:
                self._flush(batch)
                batch, acc = [], 0
            batch.append(f)
            acc += f[4]
        self._flush(batch)

    def _flush(self, batch) -> None:
        if not batch:
            return
        streams, crcs = self._r._read_deflate([f[3] for f in batch], [f[4] for f in batch], True, None, self._lzc)
        for (path, mode, mtime, _, size), s, c in zip(batch, streams, crcs):
            self._entry(path, mode, mtime, 8, [s], c, len(s), size)

    def _large(self, path: str, mode: int, mtime: int, payload_offset: int, size: int) -> None:
        if self._r.ReadAt(payload_offset, 16) != payload_header(size):
            raise IOError(f"transfer: file at payload offset {payload_offset} ({size} bytes): DEC_BAD_HEADER")

        # the local header carries no CRC or sizes (flag bit 3): the pieces stream out, then the descriptor
        e = _engine.zip_entry(path.encode(), mode, int(mtime), 8, 0, 0, size, self._pos)
        self._write(_engine.zip_local_header(e))
        lo, crc, csize = 0, 0, 0
        while lo < size:
            n = min(self._piece, size - lo)
            (s,), (c,) = self._r._read_deflate([payload_offset + 16 + lo], [n], False, [int(lo + n < size)], self._lzc)
            crc, csize, lo = _engine.crc32_combine(crc, c, n), csize + len(s), lo + n
            self._write(s)
        e.crc, e.comp_size = crc, csize
        self._write(_engine.zip_data_descriptor(e))
        self._entries.append(e)

    def Close(self) -> None:
        self._write(_engine.zip_directory(self._entries, self._pos))


def NewRemoteDedupSplitArchiveWriter(engine: Engine, config: Cfg, known: DigestSet | None = None,
                                     orig_payload_idx: bytes | None = None, upload=None, upload_blob=None) -> DedupWriter:
    """commit.go:329.  `orig_payload_idx` = bytes of the previous .ppxar.didx (commit.go:324-328):
    its digests seed the known set, so unchanged chunks are not uploaded again."""
    if orig_payload_idx:
        if known is None:
            known = engine.digest_set()
        known.seed_didx(orig_payload_idx)
    return DedupWriter(engine, config, known, upload, upload_blob)


def verifyBackedFileHashes(engine: Engine, open_file: Callable[[str], BinaryIO], hashes: dict[str, int],
                           batch_bytes: int = 1 << 30) -> None:
    """Mirror of verifyBackedFileHashes (reference internal/pxarmount/commit.go:957-976): every backed file is read
    again and its XXH3-64 must equal the value recorded at upload time.  The reference hashes on the host through a
    64 KiB copy buffer, one file at a time; here the files are packed into batches and hashed by ONE
    pbsgpu_xxh3_batch call each.  Errors keep the reference's wording:
    `open backed file "<p>" for verification: ...` and `backed file "<p>" content hash differs`."""
    names: list[str] = []
    arrs: list[np.ndarray] = []
    held = 0

    def flush() -> None:
        nonlocal names, arrs, held
        if not names:
            return
        got = engine.xxh3_batch(*_engine._pack(arrs))
        for name, h in zip(names, got):
            if int(h) != hashes[name]:
                raise IOError(f'backed file "{name}" content hash differs')
        names, arrs, held = [], [], 0

    for rel in hashes:
        try:
            with open_file(rel) as f:
                data = f.read()
        except OSError as ex:
            raise IOError(f'open backed file "{rel}" for verification: {ex}') from ex
        names.append(rel)
        arrs.append(np.frombuffer(data, dtype=np.uint8))
        held += len(data)
        if held >= batch_bytes:
            flush()
    flush()
