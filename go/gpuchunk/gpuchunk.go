//go:build gpu && cgo

// Package gpuchunk is the cgo shim a pbs-plus maintainer adds to call libpbsgpu.so
// (include/pbsgpu.h) from the Go host code.  It is the reference-side binding for the
// ONE hot path this repository accelerates: buzhash boundary scan + per-chunk SHA-256 +
// known-digest probe, i.e. what happens inside
//
//	writer.WriteEntryReader(entry, tee, size)          internal/pxarmount/commit.go:720, :858
//
// configured by buzhash.NewConfig(4096) (commit.go:302-305) and seeded from the previous
// snapshot's index (commit.go:286-294, :324-329).
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain (SURVEY.md
// section 0).  The same C symbols are exercised by the Python ctypes tests (tests/) and the
// C++ driver (tests/cxx/).  pxar-mount is built CGO_ENABLED=0 today (.goreleaser.yaml:56);
// this file only builds with `-tags gpu` and CGO_ENABLED=1.
package gpuchunk

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../pbs_plus_b200 -lpbsgpu -Wl,-rpath,${SRCDIR}/../../pbs_plus_b200
#include <stdlib.h>
#include "pbsgpu.h"
*/
import "C"

import (
	"bytes"
	"crypto/rand"
	"errors"
	"fmt"
	"hash/crc32"
	"io"
	"os"
	"runtime"
	"strings"
	"time"
	"unsafe"
)

// Config mirrors buzhash.Config (opaque in the reference; built by NewConfig).
type Config struct{ c C.pbsgpu_cfg }

// NewConfig mirrors buzhash.NewConfig(avgKiB) (commit.go:303 passes 4096 = 4 MiB).
func NewConfig(avgKiB int) (Config, error) {
	var cfg Config
	if rc := C.pbsgpu_config_kib(C.uint32_t(avgKiB), nil, &cfg.c); rc != 0 {
		return cfg, fmt.Errorf("buzhash: invalid average chunk size %d KiB (rc %d)", avgKiB, int(rc))
	}
	return cfg, nil
}

// Engine is one GPU context.  Safe to use from any goroutine: the C side binds the device
// per call and serialises calls per context (no thread-local CUDA state).
type Engine struct{ ctx *C.pbsgpu_ctx }

func Open(device int) (*Engine, error) {
	var ctx *C.pbsgpu_ctx
	if rc := C.pbsgpu_open(C.int(device), &ctx); rc != 0 {
		return nil, fmt.Errorf("pbsgpu_open(%d): rc %d (no CUDA device; there is no CPU fallback)", device, int(rc))
	}
	e := &Engine{ctx}
	runtime.SetFinalizer(e, func(e *Engine) { e.Close() })
	return e, nil
}

func (e *Engine) Close() {
	if e.ctx != nil {
		C.pbsgpu_close(e.ctx)
		e.ctx = nil
	}
}

func (e *Engine) err(rc C.int) error {
	if rc == 0 {
		return nil
	}
	return fmt.Errorf("pbsgpu: %s (rc %d)", C.GoString(C.pbsgpu_strerror(e.ctx)), int(rc))
}

// KnownSet mirrors the session's known-chunk bookkeeping (PreviousBackupRef, commit.go:286-294).
type KnownSet struct {
	e *Engine
	s *C.pbsgpu_set
}

func (e *Engine) NewKnownSet(capacityHint uint64) (*KnownSet, error) {
	var s *C.pbsgpu_set
	if err := e.err(C.pbsgpu_set_create(e.ctx, C.uint64_t(capacityHint), &s)); err != nil {
		return nil, err
	}
	return &KnownSet{e, s}, nil
}

// SeedFromDidx feeds the bytes of the previous .ppxar.didx (origPayloadIdx, commit.go:324-328).
func (k *KnownSet) SeedFromDidx(didx []byte) (uint64, error) {
	if len(didx) == 0 {
		return 0, nil
	}
	var n C.uint64_t
	rc := C.pbsgpu_set_seed_didx(k.s, (*C.uint8_t)(unsafe.Pointer(&didx[0])), C.uint64_t(len(didx)), &n)
	return uint64(n), k.e.err(rc)
}

func (k *KnownSet) Close() { C.pbsgpu_set_destroy(k.s) }

// Chunk is one dynamic-index entry: (end offset, digest) + whether the digest was known.
type Chunk struct {
	Stream uint32
	Known  bool
	End    uint64
	Digest [32]byte
}

// ErrStagingFull is returned by WriteEntryReader when the pinned staging buffer cannot take the entry NOW:
// Flush the batch and write the entry again.
var ErrStagingFull = errors.New("pbsgpu: staging full, call Flush first")

// ErrEntryTooLarge is returned when the entry alone exceeds the staging buffer: flushing cannot help, the entry has
// to go through a Stream / PayloadWriter (which have no size limit).
var ErrEntryTooLarge = errors.New("pbsgpu: entry larger than the staging buffer, use a Stream")

// Batch accumulates whole files in C-owned PINNED staging (Go pointers are never retained by C)
// and pushes them through the GPU in one call -- the batched form of the per-file loop at
// commit.go:604-625 / :697-731.
type Batch struct {
	e    *Engine
	cfg  Config
	buf  unsafe.Pointer
	cap  uint64
	fill uint64
	off  []C.uint64_t
	ln   []C.uint64_t
}

func (e *Engine) NewBatch(cfg Config, stagingBytes uint64) (*Batch, error) {
	p := C.pbsgpu_host_alloc(e.ctx, C.uint64_t(stagingBytes))
	if p == nil {
		return nil, errors.New("pbsgpu: pinned staging allocation failed")
	}
	return &Batch{e: e, cfg: cfg, buf: p, cap: stagingBytes}, nil
}

// WriteEntryReader mirrors transfer.ArchiveWriter.WriteEntryReader(entry, reader, size): it pulls
// exactly size bytes from r (io.ReadFull semantics) into the staging buffer.
func (b *Batch) WriteEntryReader(r io.Reader, size uint64) error {
	if size > b.cap {
		return ErrEntryTooLarge
	}
	start := (b.fill + 255) &^ 255
	if start+size > b.cap {
		return ErrStagingFull
	}
	dst := unsafe.Slice((*byte)(unsafe.Add(b.buf, start)), size)
	if _, err := io.ReadFull(r, dst); err != nil {
		return fmt.Errorf("read payload: %w", err)
	}
	b.off = append(b.off, C.uint64_t(start))
	b.ln = append(b.ln, C.uint64_t(size))
	b.fill = start + size
	return nil
}

// Flush runs scan -> cut -> SHA-256 -> probe for every queued file and returns the chunks in
// (file, offset) order; Known chunks need no upload ("Only new chunks are uploaded").
func (b *Batch) Flush(known *KnownSet) ([]Chunk, error) {
	res, _, err := b.flush(known, false)
	return res, err
}

// FlushWithHashes is Flush plus the XXH3-64 (seed 0) of every queued file, computed on the GPU from the
// same staged bytes: the value emitBackedFile gets from `h := xxh3.New(); io.TeeReader(f, h); h.Sum64()`
// (commit.go:717-725) and stores in ow.backedHashes -- so the host no longer hashes while it reads.
func (b *Batch) FlushWithHashes(known *KnownSet) ([]Chunk, []uint64, error) {
	return b.flush(known, true)
}

func (b *Batch) flush(known *KnownSet, withHashes bool) ([]Chunk, []uint64, error) {
	n := len(b.off)
	if n == 0 {
		return nil, nil, nil
	}
	capChunks := uint64(n)
	for _, l := range b.ln {
		capChunks += uint64(l) / uint64(b.cfg.c.min)
	}
	out := make([]C.pbsgpu_chunk, capChunks+1)
	var nOut C.uint64_t
	var set *C.pbsgpu_set
	if known != nil {
		set = known.s
	}
	var hashes []C.uint64_t
	var hp *C.uint64_t
	if withHashes {
		hashes = make([]C.uint64_t, n)
		hp = &hashes[0]
	}
	rc := C.pbsgpu_chunk_digest_batch_xxh3(b.e.ctx, &b.cfg.c, b.buf, &b.off[0], &b.ln[0], C.uint32_t(n), set,
		&out[0], C.uint64_t(len(out)), &nOut, hp)
	if err := b.e.err(rc); err != nil {
		return nil, nil, err
	}
	res := make([]Chunk, int(nOut))
	for i := range res {
		res[i].Stream = uint32(out[i].stream)
		res[i].Known = out[i].flags&C.PBSGPU_CHUNK_KNOWN != 0
		res[i].End = uint64(out[i].end_off)
		copy(res[i].Digest[:], C.GoBytes(unsafe.Pointer(&out[i].digest[0]), 32))
	}
	var hs []uint64
	if withHashes {
		hs = make([]uint64, n)
		for i := range hashes {
			hs[i] = uint64(hashes[i])
		}
	}
	b.off, b.ln, b.fill = b.off[:0], b.ln[:0], 0
	return res, hs, nil
}

// FileHashes returns the XXH3-64 of every queued file WITHOUT chunking: the verify pass of the commit
// (verifyBackedFileHashes, commit.go:957-976) re-reads the backed files into the staging buffer with
// WriteEntryReader and compares these values with ow.backedHashes.  The queue is cleared.
func (b *Batch) FileHashes() ([]uint64, error) {
	n := len(b.off)
	if n == 0 {
		return nil, nil
	}
	hashes := make([]C.uint64_t, n)
	rc := C.pbsgpu_xxh3_batch(b.e.ctx, b.buf, &b.off[0], &b.ln[0], C.uint32_t(n), &hashes[0])
	if err := b.e.err(rc); err != nil {
		return nil, err
	}
	res := make([]uint64, n)
	for i := range hashes {
		res[i] = uint64(hashes[i])
	}
	b.off, b.ln, b.fill = b.off[:0], b.ln[:0], 0
	return res, nil
}

func (b *Batch) Close() { C.pbsgpu_host_free(b.e.ctx, b.buf) }

// BuildDidx renders the dynamic-index image (<name>.ppxar.didx, commit.go:321-322) for chunks in
// (stream, offset) order; offsets are cumulative over the archive stream, the checksum is computed on the GPU.
func (e *Engine) BuildDidx(chunks []Chunk, uuid [16]byte, ctime int64) ([]byte, error) {
	n := len(chunks)
	rec := make([]C.pbsgpu_chunk, n+1)
	for i, c := range chunks {
		rec[i].stream = C.uint32_t(c.Stream)
		rec[i].end_off = C.uint64_t(c.End)
		for k := 0; k < 32; k++ {
			rec[i].digest[k] = C.uint8_t(c.Digest[k])
		}
	}
	out := make([]byte, uint64(C.pbsgpu_didx_size(C.uint64_t(n))))
	rc := C.pbsgpu_didx_build(e.ctx, &rec[0], C.uint64_t(n), (*C.uint8_t)(unsafe.Pointer(&uuid[0])), C.int64_t(ctime),
		(*C.uint8_t)(unsafe.Pointer(&out[0])), C.uint64_t(len(out)))
	return out, e.err(rc)
}

// BlobCRC32 returns the DataBlob payload checksums of ranges [off[i], off[i]+len[i]) of the batch's pinned
// staging buffer (only NEW chunks need a blob; POST /dynamic_chunk).
func (b *Batch) BlobCRC32(off, length []uint64) ([]uint32, error) {
	n := len(off)
	if n == 0 {
		return nil, nil
	}
	o := make([]C.uint64_t, n)
	l := make([]C.uint64_t, n)
	for i := range off {
		o[i], l[i] = C.uint64_t(off[i]), C.uint64_t(length[i])
	}
	crc := make([]C.uint32_t, n)
	rc := C.pbsgpu_crc32_batch(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), &crc[0])
	if err := b.e.err(rc); err != nil {
		return nil, err
	}
	res := make([]uint32, n)
	for i := range crc {
		res[i] = uint32(crc[i])
	}
	return res, nil
}

// ---------------------------------------------------------------------------------------------------------------
// Streaming form: ONE byte stream of any length (a VM image, or the whole pxar payload stream), state carried
// across writes -- the literal drop-in for writer.WriteEntryReader(entry, io.Reader, size) (commit.go:718-720).
// ---------------------------------------------------------------------------------------------------------------

// Stream wraps pbsgpu_stream_*.  Bytes travel through a pinned staging ring owned by the C side (reserve -> the
// reader fills it -> commit starts the DMA); Go memory is never retained by C.
type Stream struct {
	e *Engine
	s *C.pbsgpu_stream
}

func (e *Engine) NewStream(cfg Config, known *KnownSet) (*Stream, error) {
	var set *C.pbsgpu_set
	if known != nil {
		set = known.s
	}
	var s *C.pbsgpu_stream
	if err := e.err(C.pbsgpu_stream_open(e.ctx, &cfg.c, set, &s)); err != nil {
		return nil, err
	}
	return &Stream{e, s}, nil
}

// ReadFrom pulls exactly size bytes from r straight into the pinned ring (io.ReadFull per slot), no intermediate copy.
func (st *Stream) ReadFrom(r io.Reader, size uint64) error {
	slot := uint64(C.pbsgpu_stream_slot_bytes(st.s))
	for size > 0 {
		var p unsafe.Pointer
		if err := st.e.err(C.pbsgpu_stream_reserve(st.s, &p)); err != nil {
			return err
		}
		n := size
		if n > slot {
			n = slot
		}
		if _, err := io.ReadFull(r, unsafe.Slice((*byte)(p), n)); err != nil {
			C.pbsgpu_stream_commit(st.s, 0)
			return fmt.Errorf("read payload: %w", err)
		}
		if err := st.e.err(C.pbsgpu_stream_commit(st.s, C.uint64_t(n))); err != nil {
			return err
		}
		size -= n
	}
	return nil
}

// Write implements io.Writer (pageable Go memory is copied into the ring slot by slot).
func (st *Stream) Write(p []byte) (int, error) {
	if len(p) == 0 {
		return 0, nil
	}
	if err := st.e.err(C.pbsgpu_stream_write(st.s, unsafe.Pointer(&p[0]), C.uint64_t(len(p)))); err != nil {
		return 0, err
	}
	return len(p), nil
}

// Suggest registers a suggested boundary at the CURRENT position (call it right before writing a file's PAYLOAD header).
func (st *Stream) Suggest() error {
	return st.e.err(C.pbsgpu_stream_suggest(st.s, C.pbsgpu_stream_position(st.s)))
}

func (st *Stream) Position() uint64 { return uint64(C.pbsgpu_stream_position(st.s)) }

// Poll returns the chunks finished so far (stream order); Finish flushes the final short chunk first.
func (st *Stream) Poll() ([]Chunk, error) {
	var all []Chunk
	buf := make([]C.pbsgpu_chunk, 4096)
	for {
		var n C.uint64_t
		if err := st.e.err(C.pbsgpu_stream_poll(st.s, &buf[0], C.uint64_t(len(buf)), &n)); err != nil {
			return all, err
		}
		if n == 0 {
			return all, nil
		}
		for i := 0; i < int(n); i++ {
			var c Chunk
			c.Known = buf[i].flags&C.PBSGPU_CHUNK_KNOWN != 0
			c.End = uint64(buf[i].end_off)
			copy(c.Digest[:], C.GoBytes(unsafe.Pointer(&buf[i].digest[0]), 32))
			all = append(all, c)
		}
	}
}

func (st *Stream) Finish() ([]Chunk, error) {
	if err := st.e.err(C.pbsgpu_stream_finish(st.s)); err != nil {
		return nil, err
	}
	return st.Poll()
}

func (st *Stream) Close() { C.pbsgpu_stream_close(st.s) }

// Blob modes of SetBlobMode: the encoders of Batch.BlobEncode, BlobEncodeZ, BlobEncodeLZ, BlobEncodeLZE,
// BlobEncodeLZH, BlobEncodeLZL (its value is 7) and BlobEncodeLZC (10; 6, 8 and 9 are not assigned).
const (
	BlobNone = C.PBSGPU_BLOB_NONE
	BlobRaw  = C.PBSGPU_BLOB_RAW
	BlobZ    = C.PBSGPU_BLOB_Z
	BlobLZ   = C.PBSGPU_BLOB_LZ
	BlobLZE  = C.PBSGPU_BLOB_LZE
	BlobLZH  = C.PBSGPU_BLOB_LZH
	BlobLZL  = C.PBSGPU_BLOB_LZL
	BlobLZC  = C.PBSGPU_BLOB_LZC
)

// SetBlobMode makes the stream encode a DataBlob for every new chunk on the GPU (before the first byte).
func (st *Stream) SetBlobMode(mode int) error { return st.e.err(C.pbsgpu_stream_blob_mode(st.s, C.int(mode))) }

// PollBlobs returns up to max blobs available now; blob k belongs to the k-th chunk without Known in Poll order.
func (st *Stream) PollBlobs(buf []byte, max int) ([][]byte, error) {
	var out [][]byte
	lens := make([]C.uint64_t, 256)
	for len(out) < max {
		want := max - len(out)
		if want > len(lens) {
			want = len(lens)
		}
		var n C.uint64_t
		if err := st.e.err(C.pbsgpu_stream_poll_blobs(st.s, (*C.uint8_t)(unsafe.Pointer(&buf[0])), C.uint64_t(len(buf)),
			&lens[0], C.uint64_t(want), &n)); err != nil {
			return out, err
		}
		if n == 0 {
			break
		}
		pos := uint64(0)
		for i := 0; i < int(n); i++ {
			out = append(out, append([]byte(nil), buf[pos:pos+uint64(lens[i])]...))
			pos += uint64(lens[i])
		}
	}
	return out, nil
}

// HashRange registers [offset, offset+length) for XXH3-64 before its bytes are written.
func (st *Stream) HashRange(offset, length uint64) error {
	return st.e.err(C.pbsgpu_stream_hash_range(st.s, C.uint64_t(offset), C.uint64_t(length)))
}

// PollHashes returns the hashes of the registered ranges available now, in registration order.
func (st *Stream) PollHashes() ([]uint64, error) {
	var all []uint64
	buf := make([]C.uint64_t, 4096)
	for {
		var n C.uint64_t
		if err := st.e.err(C.pbsgpu_stream_poll_hashes(st.s, &buf[0], C.uint64_t(len(buf)), &n)); err != nil {
			return all, err
		}
		if n == 0 {
			return all, nil
		}
		for i := 0; i < int(n); i++ {
			all = append(all, uint64(buf[i]))
		}
	}
}

// PayloadWriter produces the pxar v2 PAYLOAD stream the production chunker sees -- start marker, then per file a
// 16-byte PAYLOAD header + content (internal/pxarmount/pxarfs.go:408-411) -- through ONE Stream, with a suggested
// boundary at every file start.  WriteEntryReader returns the entry's payload offset (what the mpxar PAYLOAD_REF
// stores).  This, not per-file batching, is the layout an existing .ppxar.didx describes.
//
// With PayloadOptions.BlobMode set, UploadBlob receives the DataBlob of every new chunk (encoded on the GPU from the
// stream's windows: "upload only !Known chunks"); with HashFiles, BackedHashes maps each path to the file's XXH3-64
// (commitWalkState.backedHashes, commit.go:725).
type PayloadWriter struct {
	st           *Stream
	Chunks       []Chunk
	started      bool
	opt          PayloadOptions
	blobBuf      []byte
	pending      []Digest // digests of new chunks whose blob has not come back yet
	hashed       []string // paths whose hash has not come back yet
	BackedHashes map[string]uint64
}

type PayloadOptions struct {
	BlobMode   int
	UploadBlob func(digest Digest, blob []byte) error
	HashFiles  bool
	Crypt      *Crypt // encrypt mode: keyed digests, encrypted blobs (nil: CryptModeNone)
}

const (
	pxarPayload            = 0x28147a1b0b7c1a25
	pxarPayloadStartMarker = 0x834c68c2194a4ed2
	pxarPayloadTailMarker  = 0x6c72b78b984c81b5
)

func header(htype, fullSize uint64) []byte {
	var h [16]byte
	for i := 0; i < 8; i++ {
		h[i] = byte(htype >> (8 * i))
		h[8+i] = byte(fullSize >> (8 * i))
	}
	return h[:]
}

func (e *Engine) NewPayloadWriter(cfg Config, known *KnownSet) (*PayloadWriter, error) {
	return e.NewPayloadWriterOpts(cfg, known, PayloadOptions{})
}

func (e *Engine) NewPayloadWriterOpts(cfg Config, known *KnownSet, opt PayloadOptions) (*PayloadWriter, error) {
	st, err := e.NewStream(cfg, known)
	if err != nil {
		return nil, err
	}
	w := &PayloadWriter{st: st, opt: opt, BackedHashes: map[string]uint64{}}
	if opt.Crypt != nil {
		if err := st.SetCrypt(opt.Crypt); err != nil {
			st.Close()
			return nil, err
		}
	}
	if opt.BlobMode != BlobNone {
		if opt.UploadBlob == nil {
			st.Close()
			return nil, fmt.Errorf("gpuchunk: a blob mode needs an UploadBlob callback")
		}
		if err := st.SetBlobMode(opt.BlobMode); err != nil {
			st.Close()
			return nil, err
		}
		w.blobBuf = make([]byte, uint64(C.pbsgpu_blob_size_enc(cfg.c.max))+16<<20)
	}
	_, err = st.Write(header(pxarPayloadStartMarker, 16))
	return w, err
}

// WriteEntryReader writes one file without a path; with HashFiles set, use WriteBackedEntry so that the hash has a key.
func (w *PayloadWriter) WriteEntryReader(r io.Reader, size uint64) (payloadOffset uint64, err error) {
	if w.opt.HashFiles {
		return 0, fmt.Errorf("gpuchunk: with HashFiles, files are written through WriteBackedEntry(path, ...)")
	}
	return w.WriteBackedEntry("", r, size)
}

// WriteBackedEntry is WriteEntryReader for the file at path (relPath in emitBackedFile): with HashFiles set, its
// XXH3-64 lands in BackedHashes[path].
func (w *PayloadWriter) WriteBackedEntry(path string, r io.Reader, size uint64) (payloadOffset uint64, err error) {
	payloadOffset = w.st.Position()
	if err = w.st.Suggest(); err != nil {
		return
	}
	if w.opt.HashFiles {
		if err = w.st.HashRange(payloadOffset+16, size); err != nil {
			return
		}
		w.hashed = append(w.hashed, path)
	}
	if _, err = w.st.Write(header(pxarPayload, 16+size)); err != nil {
		return
	}
	if err = w.st.ReadFrom(r, size); err != nil {
		return
	}
	done, err := w.st.Poll()
	if err == nil {
		err = w.drain(done)
	}
	return
}

// drain records the chunks, uploads the blobs of the new ones whose records are here and stores the finished hashes.
func (w *PayloadWriter) drain(done []Chunk) error {
	w.Chunks = append(w.Chunks, done...)
	if w.opt.BlobMode != BlobNone {
		for _, c := range done {
			if !c.Known {
				w.pending = append(w.pending, c.Digest)
			}
		}
		blobs, err := w.st.PollBlobs(w.blobBuf, len(w.pending))
		for i, b := range blobs {
			if err == nil {
				err = w.opt.UploadBlob(w.pending[i], b)
			}
		}
		w.pending = w.pending[len(blobs):]
		if err != nil {
			return err
		}
	}
	if len(w.hashed) > 0 {
		hs, err := w.st.PollHashes()
		for i, h := range hs {
			w.BackedHashes[w.hashed[i]] = h
		}
		w.hashed = w.hashed[len(hs):]
		if err != nil {
			return err
		}
	}
	return nil
}

func (w *PayloadWriter) Finish() ([]Chunk, error) {
	if _, err := w.st.Write(header(pxarPayloadTailMarker, 16)); err != nil {
		return nil, err
	}
	done, err := w.st.Finish()
	if err == nil {
		err = w.drain(done)
	}
	w.st.Close()
	return w.Chunks, err
}

// ---------------------------------------------------------------------------------------------------------------
// Multi-GPU: one Engine per GPU (one goroutine each), files sharded by range; the ONE exchange step.
// ---------------------------------------------------------------------------------------------------------------

// NcclComm is an ncclComm_t made through the C ABI's helpers; a caller with its own NCCL binding passes its
// communicator to AllGather through NcclCommFromHandle instead.
type NcclComm struct{ h unsafe.Pointer }

func NcclUniqueID() ([128]byte, error) {
	var id [128]byte
	if rc := C.pbsgpu_nccl_unique_id((*C.uint8_t)(unsafe.Pointer(&id[0]))); rc != 0 {
		return id, fmt.Errorf("pbsgpu: NCCL unavailable (rc %d)", int(rc))
	}
	return id, nil
}

func (e *Engine) NewNcclComm(id [128]byte, nranks, rank int) (*NcclComm, error) {
	var h unsafe.Pointer
	if err := e.err(C.pbsgpu_nccl_comm_create(e.ctx, (*C.uint8_t)(unsafe.Pointer(&id[0])), C.int(nranks), C.int(rank), &h)); err != nil {
		return nil, err
	}
	return &NcclComm{h}, nil
}

func NcclCommFromHandle(h unsafe.Pointer) *NcclComm { return &NcclComm{h} }
func (c *NcclComm) Close()                           { C.pbsgpu_nccl_comm_destroy(c.h) }

// AllGather merges this rank's chunk digests with every other rank's (pbsgpu_set_allgather: counts + padded
// digests over NCCL/NVLink, then every replica inserts all of them in global (rank, index) order) and sets
// Known on the chunks that are known globally.  Collective: every rank calls it once per batch.
func (k *KnownSet) AllGather(comm *NcclComm, chunks []Chunk) error {
	n := len(chunks)
	dig := make([]byte, 32*n+1)
	hit := make([]byte, n+1)
	for i := range chunks {
		copy(dig[32*i:], chunks[i].Digest[:])
	}
	rc := C.pbsgpu_set_allgather(k.s, comm.h, (*C.uint8_t)(unsafe.Pointer(&dig[0])), C.uint64_t(n), (*C.uint8_t)(unsafe.Pointer(&hit[0])))
	if err := k.e.err(rc); err != nil {
		return err
	}
	for i := range chunks {
		chunks[i].Known = hit[i] != 0
	}
	return nil
}

// BlobEncode renders complete uncompressed DataBlobs (magic | crc32 | payload) for ranges of the batch's staging
// buffer -- the upload bodies of the NEW chunks (POST /dynamic_chunk, internal/server/backup/log_cleanup.go:19-31).
func (b *Batch) BlobEncode(off, length []uint64) ([][]byte, error) {
	n := len(off)
	if n == 0 {
		return nil, nil
	}
	o := make([]C.uint64_t, n)
	l := make([]C.uint64_t, n)
	oo := make([]C.uint64_t, n)
	var total uint64
	for i := range off {
		o[i], l[i], oo[i] = C.uint64_t(off[i]), C.uint64_t(length[i]), C.uint64_t(total)
		total += uint64(C.pbsgpu_blob_size(C.uint64_t(length[i])))
	}
	out := make([]byte, total+1)
	rc := C.pbsgpu_blob_encode_batch(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), (*C.uint8_t)(unsafe.Pointer(&out[0])), &oo[0], nil)
	if err := b.e.err(rc); err != nil {
		return nil, err
	}
	res := make([][]byte, n)
	for i := range off {
		res[i] = out[uint64(oo[i]) : uint64(oo[i])+12+length[i]]
	}
	return res, nil
}

// BlobEncodeZ is BlobEncode with the zstd-compressed DataBlob form where that is smaller (upstream DataBlob::encode
// keeps a compressed payload only then).  The frames are built on the GPU from RLE and raw blocks -- they remove
// the zero runs of disk images and sparse files; data without such runs stays uncompressed.
func (b *Batch) BlobEncodeZ(off, length []uint64) ([][]byte, error) {
	return b.blobEncodeCompressed(off, length, blobZ)
}

// BlobEncodeLZ is BlobEncodeZ with a match stage: every 128 KiB block that is not one repeated byte becomes a zstd
// Compressed_Block (greedy LZ77 inside the block, raw literals, predefined FSE tables) where that is smaller, so
// text, logs and other compressible data shrink too.  Each blob is at most the size of its BlobEncodeZ blob.
func (b *Batch) BlobEncodeLZ(off, length []uint64) ([][]byte, error) {
	return b.blobEncodeCompressed(off, length, blobLZ)
}

// BlobEncodeLZE is BlobEncodeLZ with zstd's entropy stage: each compressed block is the smaller of the BlobEncodeLZ
// one and one with tables fitted to the block (FSE_Compressed_Mode sequences, Huffman literals).  Each blob is at most
// the size of its BlobEncodeLZ blob.  Like the rest of this shim, it has not been compiled against a Go toolchain.
func (b *Batch) BlobEncodeLZE(off, length []uint64) ([][]byte, error) {
	return b.blobEncodeCompressed(off, length, blobLZE)
}

// BlobEncodeLZH is BlobEncodeLZE with Huffman literals whatever their largest byte value: the tree is written in the
// direct or the FSE-compressed weight form, the smaller one, so binary data gets entropy-coded literals too.  Each blob
// is at most the size of its BlobEncodeLZE blob.  Like the rest of this shim, it has not been compiled against a Go
// toolchain.
func (b *Batch) BlobEncodeLZH(off, length []uint64) ([][]byte, error) {
	return b.blobEncodeCompressed(off, length, blobLZH)
}

// BlobEncodeLZL is BlobEncodeLZH plus long-distance matches: repeats anywhere earlier in the same chunk (a copy of a
// file inside one chunk, repeated pages of an image) become long matches of the blocks they cross, where that makes the
// block smaller.  Each blob is at most the size of its BlobEncodeLZH blob.  Like the rest of this shim, it has not been
// compiled against a Go toolchain.
func (b *Batch) BlobEncodeLZL(off, length []uint64) ([][]byte, error) {
	return b.blobEncodeCompressed(off, length, blobLZL)
}

// BlobEncodeLZC is BlobEncodeLZH with a stronger match search: the longest of the 16 latest earlier positions of the
// chunk with the same 4 bytes, up to 2^24 - 4 bytes back, and a lazy parse.  Text-like chunks get smaller blobs for more
// GPU time; ranges must be shorter than 2^32 bytes.  Like the rest of this shim, it has not been compiled against a Go
// toolchain.
func (b *Batch) BlobEncodeLZC(off, length []uint64) ([][]byte, error) {
	return b.blobEncodeCompressed(off, length, blobLZC)
}

// which compressed DataBlob encoder blobEncodeCompressed calls
type blobMode int

const (
	blobZ blobMode = iota
	blobLZ
	blobLZE
	blobLZH
	blobLZL
	blobLZC
)

func (b *Batch) blobEncodeCompressed(off, length []uint64, mode blobMode) ([][]byte, error) {
	n := len(off)
	if n == 0 {
		return nil, nil
	}
	o := make([]C.uint64_t, n)
	l := make([]C.uint64_t, n)
	oo := make([]C.uint64_t, n)
	ol := make([]C.uint64_t, n)
	var total uint64
	for i := range off {
		o[i], l[i], oo[i] = C.uint64_t(off[i]), C.uint64_t(length[i]), C.uint64_t(total)
		total += uint64(C.pbsgpu_blob_size(C.uint64_t(length[i])))
	}
	out := make([]byte, total+1)
	dst := (*C.uint8_t)(unsafe.Pointer(&out[0]))
	var rc C.int
	switch mode {
	case blobLZC:
		rc = C.pbsgpu_blob_encode_batch_lzc(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), dst, &oo[0], &ol[0], nil)
	case blobLZL:
		rc = C.pbsgpu_blob_encode_batch_lzl(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), dst, &oo[0], &ol[0], nil)
	case blobLZH:
		rc = C.pbsgpu_blob_encode_batch_lzh(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), dst, &oo[0], &ol[0], nil)
	case blobLZE:
		rc = C.pbsgpu_blob_encode_batch_lze(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), dst, &oo[0], &ol[0], nil)
	case blobLZ:
		rc = C.pbsgpu_blob_encode_batch_lz(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), dst, &oo[0], &ol[0], nil)
	default:
		rc = C.pbsgpu_blob_encode_batch_z(b.e.ctx, b.buf, &o[0], &l[0], C.uint32_t(n), dst, &oo[0], &ol[0], nil)
	}
	if err := b.e.err(rc); err != nil {
		return nil, err
	}
	res := make([][]byte, n)
	for i := range off {
		res[i] = out[uint64(oo[i]) : uint64(oo[i])+uint64(ol[i])]
	}
	return res, nil
}

// BlobDecode checks, decodes and verifies unencrypted DataBlobs (pbsgpu_blob_decode_batch): what a restore, a mount
// with --verify-chunks or a verify job does per chunk.  blobs are the blobs as read from the datastore; chunkLen and
// digests come from the dynamic index (the difference of consecutive end offsets, and each entry's digest; nil digests:
// no digest check).  wantData false is verify only: no decoded byte leaves the GPU.  Returns one PBSGPU_DEC_* status
// per blob (0 = OK) and, with wantData, the chunks whose status is OK or BAD_DIGEST.
func (e *Engine) BlobDecode(blobs [][]byte, chunkLen []uint64, digests [][32]byte, wantData bool) ([]int32, [][]byte, error) {
	return e.blobDecode(nil, blobs, chunkLen, digests, wantData)
}

// BlobDecodeEnc is BlobDecode for a snapshot written in encrypt mode (pbsgpu_blob_decode_batch_enc): encrypted blobs
// are decrypted with c's key once their AES-256-GCM tag verified (PBSGPU_DEC_BAD_TAG otherwise), and their digests are
// the keyed ones of the index (SHA-256(chunk || id_key)); unencrypted blobs are read as BlobDecode reads them.
func (e *Engine) BlobDecodeEnc(c *Crypt, blobs [][]byte, chunkLen []uint64, digests [][32]byte, wantData bool) ([]int32, [][]byte, error) {
	if c == nil {
		return nil, nil, fmt.Errorf("pbsgpu: BlobDecodeEnc needs a crypt handle")
	}
	return e.blobDecode(c, blobs, chunkLen, digests, wantData)
}

func (e *Engine) blobDecode(c *Crypt, blobs [][]byte, chunkLen []uint64, digests [][32]byte, wantData bool) ([]int32, [][]byte, error) {
	n := len(blobs)
	if n == 0 {
		return nil, nil, nil
	}
	var total, out uint64
	o := make([]C.uint64_t, n)
	l := make([]C.uint64_t, n)
	cl := make([]C.uint64_t, n)
	oo := make([]C.uint64_t, n)
	for i, b := range blobs {
		o[i], l[i], cl[i], oo[i] = C.uint64_t(total), C.uint64_t(len(b)), C.uint64_t(chunkLen[i]), C.uint64_t(out)
		total += uint64(len(b))
		out += chunkLen[i]
	}
	src := make([]byte, total+1)
	for i, b := range blobs {
		copy(src[uint64(o[i]):], b)
	}
	var dig *C.uint8_t
	if digests != nil {
		dig = (*C.uint8_t)(unsafe.Pointer(&digests[0][0]))
	}
	var dst []byte
	var dstp *C.uint8_t
	if wantData {
		dst = make([]byte, out+1)
		dstp = (*C.uint8_t)(unsafe.Pointer(&dst[0]))
	}
	status := make([]int32, n)
	var rc C.int
	if c == nil {
		rc = C.pbsgpu_blob_decode_batch(e.ctx, unsafe.Pointer(&src[0]), &o[0], &l[0], C.uint32_t(n), &cl[0], dig, dstp, &oo[0],
			(*C.int32_t)(unsafe.Pointer(&status[0])), nil)
	} else {
		rc = C.pbsgpu_blob_decode_batch_enc(e.ctx, c.c, unsafe.Pointer(&src[0]), &o[0], &l[0], C.uint32_t(n), &cl[0], dig, dstp,
			&oo[0], (*C.int32_t)(unsafe.Pointer(&status[0])), nil)
	}
	if err := e.err(rc); err != nil {
		return nil, nil, err
	}
	if !wantData {
		return status, nil, nil
	}
	res := make([][]byte, n)
	for i := range blobs {
		if status[i] == int32(C.PBSGPU_DEC_OK) || status[i] == int32(C.PBSGPU_DEC_BAD_DIGEST) {
			res[i] = dst[uint64(oo[i]) : uint64(oo[i])+chunkLen[i]]
		}
	}
	return status, res, nil
}

// Crypt is one 32-byte client key of encrypt mode (BackupConfig's CryptMode, commit.go:314) on the engine's device.
type Crypt struct{ c *C.pbsgpu_crypt }

func (e *Engine) NewCrypt(key [32]byte) (*Crypt, error) {
	var c *C.pbsgpu_crypt
	if err := e.err(C.pbsgpu_crypt_create(e.ctx, (*C.uint8_t)(unsafe.Pointer(&key[0])), &c)); err != nil {
		return nil, err
	}
	return &Crypt{c}, nil
}

// Close zeroes the key material on the host and the device.
func (c *Crypt) Close() { C.pbsgpu_crypt_destroy(c.c) }

// SetCrypt puts the stream in encrypt mode (before the first byte): keyed digests, and encrypted blobs whose IVs the
// library draws from the OS CSPRNG.
func (st *Stream) SetCrypt(c *Crypt) error { return st.e.err(C.pbsgpu_stream_crypt(st.s, c.c, nil)) }

// BlobEncodeEnc returns encrypted DataBlobs of the ranges: mode (BlobRaw .. BlobLZH, BlobLZL, BlobLZC) picks the compressor whose frame
// is encrypted when smaller.  Every blob gets a fresh IV from crypto/rand; an IV must never repeat under one key.
func (b *Batch) BlobEncodeEnc(c *Crypt, mode int, off, length []uint64) ([][]byte, error) {
	n := len(off)
	if n == 0 {
		return nil, nil
	}
	iv := make([]byte, 16*n)
	if _, err := rand.Read(iv); err != nil {
		return nil, err
	}
	o := make([]C.uint64_t, n)
	l := make([]C.uint64_t, n)
	oo := make([]C.uint64_t, n)
	ol := make([]C.uint64_t, n)
	var total uint64
	for i := range off {
		o[i], l[i], oo[i] = C.uint64_t(off[i]), C.uint64_t(length[i]), C.uint64_t(total)
		total += uint64(C.pbsgpu_blob_size_enc(C.uint64_t(length[i])))
	}
	out := make([]byte, total+1)
	rc := C.pbsgpu_blob_encode_batch_enc(b.e.ctx, c.c, C.int(mode), b.buf, &o[0], &l[0], C.uint32_t(n),
		(*C.uint8_t)(unsafe.Pointer(&iv[0])), (*C.uint8_t)(unsafe.Pointer(&out[0])), &oo[0], &ol[0], nil)
	if err := b.e.err(rc); err != nil {
		return nil, err
	}
	res := make([][]byte, n)
	for i := range off {
		res[i] = out[uint64(oo[i]) : uint64(oo[i])+uint64(ol[i])]
	}
	return res, nil
}

// PayloadReader reads a payload archive through its .ppxar.didx (pbsgpu_reader_*): the replacement for
// reader.PayloadReaderAt() that PxarFS.readFileContent calls (internal/pxarmount/pxarfs.go:38, :409-412).  Chunks are
// decoded and verified on the GPU once (CRC, GCM tag with a crypt, zstd, digest against the index) into a device cache
// of cacheBytes (0 = 256 MiB); reads are copied out of that cache.  source returns a chunk's DataBlob by digest
// (.chunks/<hex>).  Prefetch: the number of chunks after the last touched one fetched along with a miss.
type PayloadReader struct {
	e        *Engine
	r        *C.pbsgpu_reader
	source   func([32]byte) ([]byte, error)
	digests  [][32]byte
	size     uint64
	Prefetch int
}

func (e *Engine) NewPayloadReader(didx []byte, c *Crypt, cacheBytes uint64, source func([32]byte) ([]byte, error)) (*PayloadReader, error) {
	if len(didx) == 0 {
		return nil, fmt.Errorf("pbsgpu: empty index image")
	}
	var cr *C.pbsgpu_crypt
	if c != nil {
		cr = c.c
	}
	var r *C.pbsgpu_reader
	if err := e.err(C.pbsgpu_reader_open(e.ctx, (*C.uint8_t)(unsafe.Pointer(&didx[0])), C.uint64_t(len(didx)), cr,
		C.uint64_t(cacheBytes), &r)); err != nil {
		return nil, err
	}
	n := (len(didx) - 4096) / 40
	dg := make([][32]byte, n)
	for i := range dg {
		copy(dg[i][:], didx[4096+40*i+8:4096+40*i+40])
	}
	return &PayloadReader{e: e, r: r, source: source, digests: dg, size: uint64(C.pbsgpu_reader_size(r))}, nil
}

func (p *PayloadReader) Close() { C.pbsgpu_reader_close(p.r) }

// fetch plans ranges (payload: (payload offset, file size) of files) and fetches the missing blobs (plus Prefetch
// chunks after the last one): the blobs concatenated, their offsets, lengths and chunk indices, each with one
// trailing element so the slices are never empty.
func (p *PayloadReader) fetch(off, length []uint64, flags C.uint32_t) (blobs []byte, bo, bl, need []uint64, err error) {
	o := (*C.uint64_t)(unsafe.Pointer(&off[0]))
	l := (*C.uint64_t)(unsafe.Pointer(&length[0]))
	var k C.uint64_t
	need = make([]uint64, len(p.digests))
	var np *C.uint64_t
	if len(need) > 0 {
		np = (*C.uint64_t)(unsafe.Pointer(&need[0]))
	}
	if err = p.e.err(C.pbsgpu_reader_plan(p.r, o, l, C.uint32_t(len(off)), flags, np, nil, C.uint64_t(len(need)), &k)); err != nil {
		return
	}
	need = need[:k]
	if k > 0 && flags&C.PBSGPU_READ_SPARSE == 0 { // a sparse restore must not fetch the zero chunks after its range
		for c := need[k-1] + 1; c < uint64(len(p.digests)) && c <= need[k-1]+uint64(p.Prefetch); c++ {
			need = append(need, c)
		}
	}
	bo = make([]uint64, len(need)+1)
	bl = make([]uint64, len(need)+1)
	for j, c := range need {
		b, ferr := p.source(p.digests[c])
		if ferr != nil {
			return nil, nil, nil, nil, ferr
		}
		bo[j], bl[j] = uint64(len(blobs)), uint64(len(b))
		blobs = append(blobs, b...)
	}
	blobs = append(blobs, 0)
	need = append(need, 0)
	return
}

func (p *PayloadReader) statusErr(off, length []uint64, status []int32) error {
	for i, s := range status {
		if s != int32(C.PBSGPU_DEC_OK) {
			return fmt.Errorf("pbsgpu: read of %d bytes at %d: status %d", length[i], off[i], s)
		}
	}
	return nil
}

// read serves ranges into out at outOff: one plan, one fetch, one read.
func (p *PayloadReader) read(off, length []uint64, payload bool, out []byte, outOff []uint64) error {
	n := len(off)
	if n == 0 {
		return nil
	}
	var flags C.uint32_t
	if payload {
		flags = C.PBSGPU_READ_PAYLOAD
	}
	blobs, bo, bl, need, err := p.fetch(off, length, flags)
	if err != nil {
		return err
	}
	status := make([]int32, n)
	rc := C.pbsgpu_reader_read(p.r, (*C.uint64_t)(unsafe.Pointer(&off[0])), (*C.uint64_t)(unsafe.Pointer(&length[0])),
		C.uint32_t(n), flags, unsafe.Pointer(&blobs[0]), (*C.uint64_t)(unsafe.Pointer(&bo[0])),
		(*C.uint64_t)(unsafe.Pointer(&bl[0])), (*C.uint64_t)(unsafe.Pointer(&need[0])), C.uint32_t(len(need)-1),
		(*C.uint8_t)(unsafe.Pointer(&out[0])), (*C.uint64_t)(unsafe.Pointer(&outOff[0])), (*C.int32_t)(unsafe.Pointer(&status[0])), nil)
	if err := p.e.err(rc); err != nil {
		return err
	}
	return p.statusErr(off, length, status)
}

// readDeflate is read whose outputs are the ranges' raw Deflate streams, compressed on the GPU
// (pbsgpu_reader_read_deflate); more[i] != 0: a later call continues stream i; lzc: the hash-chain parse
// (PBSGPU_READ_DEFLATE_LZC).  Returns the streams and CRC-32s.
func (p *PayloadReader) readDeflate(off, length []uint64, payload bool, more []uint8, lzc bool) ([][]byte, []uint32, error) {
	n := len(off)
	if n == 0 {
		return nil, nil, nil
	}
	var flags C.uint32_t
	if payload {
		flags = C.PBSGPU_READ_PAYLOAD
	}
	blobs, bo, bl, need, err := p.fetch(off, length, flags)
	if err != nil {
		return nil, nil, err
	}
	oo := make([]uint64, n)
	var total uint64
	for i, s := range length {
		oo[i] = total
		total += uint64(C.pbsgpu_deflate_bound(C.uint64_t(s)))
	}
	out := make([]byte, total+1)
	olen := make([]uint64, n)
	crc := make([]uint32, n)
	status := make([]int32, n)
	var mp *C.uint8_t
	if more != nil {
		mp = (*C.uint8_t)(unsafe.Pointer(&more[0]))
	}
	if lzc {
		flags |= C.PBSGPU_READ_DEFLATE_LZC
	}
	rc := C.pbsgpu_reader_read_deflate(p.r, (*C.uint64_t)(unsafe.Pointer(&off[0])), (*C.uint64_t)(unsafe.Pointer(&length[0])),
		C.uint32_t(n), flags, mp, unsafe.Pointer(&blobs[0]), (*C.uint64_t)(unsafe.Pointer(&bo[0])),
		(*C.uint64_t)(unsafe.Pointer(&bl[0])), (*C.uint64_t)(unsafe.Pointer(&need[0])), C.uint32_t(len(need)-1),
		(*C.uint8_t)(unsafe.Pointer(&out[0])), (*C.uint64_t)(unsafe.Pointer(&oo[0])), (*C.uint64_t)(unsafe.Pointer(&olen[0])),
		(*C.uint32_t)(unsafe.Pointer(&crc[0])), (*C.int32_t)(unsafe.Pointer(&status[0])), nil)
	if err := p.e.err(rc); err != nil {
		return nil, nil, err
	}
	if err := p.statusErr(off, length, status); err != nil {
		return nil, nil, err
	}
	res := make([][]byte, n)
	for i := range res {
		res[i] = out[oo[i] : oo[i]+olen[i]]
	}
	return res, crc, nil
}

// ReadAt implements io.ReaderAt over the archive: short with io.EOF at its end.
func (p *PayloadReader) ReadAt(b []byte, off int64) (int, error) {
	if off < 0 {
		return 0, errors.New("pbsgpu: negative offset")
	}
	if uint64(off) >= p.size {
		return 0, io.EOF
	}
	want := uint64(len(b))
	if rest := p.size - uint64(off); want > rest {
		want = rest
	}
	if want == 0 {
		return 0, nil
	}
	if err := p.read([]uint64{uint64(off)}, []uint64{want}, false, b, []uint64{0}); err != nil {
		return 0, err
	}
	if want < uint64(len(b)) {
		return int(want), io.EOF
	}
	return int(want), nil
}

// ReadFiles returns the contents of files given by payload offset and size (restore): one read for all of them.
func (p *PayloadReader) ReadFiles(offsets, sizes []uint64) ([][]byte, error) {
	oo := make([]uint64, len(sizes))
	var total uint64
	for i, s := range sizes {
		oo[i] = total
		total += s
	}
	out := make([]byte, total+1)
	if err := p.read(offsets, sizes, true, out, oo); err != nil {
		return nil, err
	}
	res := make([][]byte, len(sizes))
	for i, s := range sizes {
		res[i] = out[oo[i] : oo[i]+s]
	}
	return res, nil
}

// SeedFromFidx feeds the previous snapshot's .fidx of the same disk image (pbsgpu_set_seed_fidx), as the upstream
// client does for fixed indexes: unchanged chunks of the image are not uploaded again.
func (k *KnownSet) SeedFromFidx(fidx []byte) (uint64, error) {
	if len(fidx) == 0 {
		return 0, fmt.Errorf("pbsgpu: empty index image")
	}
	var n C.uint64_t
	rc := C.pbsgpu_set_seed_fidx(k.s, (*C.uint8_t)(unsafe.Pointer(&fidx[0])), C.uint64_t(len(fidx)), &n)
	return uint64(n), k.e.err(rc)
}

// ImageWriter backs up a disk image as a fixed index (<name>.img.fidx; a VM disk, or
// `proxmox-backup-client backup disk.img:/dev/sdX`): the image is cut at every multiple of ChunkSize (upstream writes
// 4 MiB), read in slices of whole chunks into C-owned pinned staging, and each slice goes through the GPU in one batch
// call with fixed cuts (pbsgpu_batch_opts.fixed_size): SHA-256 per chunk (keyed with a crypt), probe against the known
// set, and, with a blob mode, the DataBlob of every new chunk handed to Upload.
type ImageWriter struct {
	e         *Engine
	known     *KnownSet
	crypt     *Crypt
	mode      int // BlobRaw .. BlobLZH, BlobLZL, BlobLZC; 0 = no blobs
	chunkSize uint64
	buf       unsafe.Pointer
	cap       uint64
	size      uint64
	ended     bool
	digests   []byte
	Upload    func(digest [32]byte, blob []byte) error
}

// NewImageWriter: chunkSize a power of two from 4 KiB to 16 MiB; stagingBytes is rounded down to whole chunks (at least
// one).  known and c may be nil; blobMode 0 encodes no blobs.
func (e *Engine) NewImageWriter(chunkSize uint32, known *KnownSet, c *Crypt, blobMode int, stagingBytes uint64) (*ImageWriter, error) {
	cs := uint64(chunkSize)
	if cs < 4096 || cs > 16<<20 || cs&(cs-1) != 0 {
		return nil, fmt.Errorf("pbsgpu: chunk size %d is not a power of two from 4 KiB to 16 MiB", cs)
	}
	stagingBytes -= stagingBytes % cs
	if stagingBytes == 0 {
		stagingBytes = cs
	}
	p := C.pbsgpu_host_alloc(e.ctx, C.uint64_t(stagingBytes))
	if p == nil {
		return nil, errors.New("pbsgpu: pinned staging allocation failed")
	}
	return &ImageWriter{e: e, known: known, crypt: c, mode: blobMode, chunkSize: cs, buf: p, cap: stagingBytes}, nil
}

// WriteFrom pulls exactly size bytes of the image from r (io.ReadFull semantics).  It may be called again for the
// bytes that follow as long as every call but the last covers whole chunks.
func (w *ImageWriter) WriteFrom(r io.Reader, size uint64) error {
	for size > 0 {
		if w.ended {
			return errors.New("pbsgpu: the image's last slice ended inside a chunk")
		}
		n := size
		if n > w.cap {
			n = w.cap
		}
		if _, err := io.ReadFull(r, unsafe.Slice((*byte)(w.buf), n)); err != nil {
			return fmt.Errorf("read image: %w", err)
		}
		if err := w.slice(n); err != nil {
			return err
		}
		size -= n
	}
	return nil
}

func (w *ImageWriter) slice(n uint64) error {
	cs := w.chunkSize
	nch := (n + cs - 1) / cs
	out := make([]C.pbsgpu_chunk, nch)
	off, ln := []C.uint64_t{0}, []C.uint64_t{C.uint64_t(n)}
	var o C.pbsgpu_batch_opts
	o.size = C.uint32_t(C.sizeof_pbsgpu_batch_opts)
	o.fixed_size = C.uint32_t(cs)
	if w.known != nil {
		o.set = w.known.s
	}
	if w.crypt != nil {
		o.crypt = w.crypt.c
	}
	var got C.uint64_t
	rc := C.pbsgpu_chunk_digest_batch_ex(w.e.ctx, nil, w.buf, &off[0], &ln[0], 1, &o, &out[0], C.uint64_t(nch), &got)
	if err := w.e.err(rc); err != nil {
		return err
	}
	var newOff, newLen []uint64
	var newDig [][32]byte
	for i := 0; i < int(got); i++ {
		var d [32]byte
		copy(d[:], C.GoBytes(unsafe.Pointer(&out[i].digest[0]), 32))
		w.digests = append(w.digests, d[:]...)
		if out[i].flags&C.PBSGPU_CHUNK_KNOWN == 0 {
			s := uint64(i) * cs
			l := cs
			if n-s < l {
				l = n - s
			}
			newOff, newLen, newDig = append(newOff, s), append(newLen, l), append(newDig, d)
		}
	}
	if w.mode != 0 && w.Upload != nil && len(newOff) > 0 {
		b := &Batch{e: w.e, buf: w.buf, cap: w.cap}
		var blobs [][]byte
		var err error
		switch {
		case w.crypt != nil:
			blobs, err = b.BlobEncodeEnc(w.crypt, w.mode, newOff, newLen)
		case w.mode == int(BlobRaw):
			blobs, err = b.BlobEncode(newOff, newLen)
		case w.mode == int(BlobZ):
			blobs, err = b.BlobEncodeZ(newOff, newLen)
		case w.mode == int(BlobLZ):
			blobs, err = b.BlobEncodeLZ(newOff, newLen)
		case w.mode == int(BlobLZE):
			blobs, err = b.BlobEncodeLZE(newOff, newLen)
		case w.mode == int(BlobLZH):
			blobs, err = b.BlobEncodeLZH(newOff, newLen)
		case w.mode == int(BlobLZC):
			blobs, err = b.BlobEncodeLZC(newOff, newLen)
		default:
			blobs, err = b.BlobEncodeLZL(newOff, newLen)
		}
		if err != nil {
			return err
		}
		for i, blob := range blobs {
			if err := w.Upload(newDig[i], blob); err != nil {
				return err
			}
		}
	}
	w.size += n
	w.ended = n%cs != 0
	return nil
}

// Finish renders the image's .fidx (checksum on the GPU).
func (w *ImageWriter) Finish(uuid [16]byte, ctime int64) ([]byte, error) {
	n := uint64(len(w.digests) / 32)
	out := make([]byte, uint64(C.pbsgpu_fidx_size(C.uint64_t(n))))
	var dp *C.uint8_t
	if n > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&w.digests[0]))
	}
	rc := C.pbsgpu_fidx_build(w.e.ctx, dp, C.uint64_t(n), C.uint64_t(w.size), C.uint64_t(w.chunkSize),
		(*C.uint8_t)(unsafe.Pointer(&uuid[0])), C.int64_t(ctime), (*C.uint8_t)(unsafe.Pointer(&out[0])), C.uint64_t(len(out)))
	if err := w.e.err(rc); err != nil {
		return nil, err
	}
	return out, nil
}

func (w *ImageWriter) Close() { C.pbsgpu_host_free(w.e.ctx, w.buf) }

// NewImageReader reads a disk image through its .fidx (pbsgpu_reader_open_fidx): the restore or map of a
// `.img.fidx` archive.  ReadAt serves byte ranges of the image; ReadFiles fails (an image has no pxar headers).
func (e *Engine) NewImageReader(fidx []byte, c *Crypt, cacheBytes uint64, source func([32]byte) ([]byte, error)) (*PayloadReader, error) {
	if len(fidx) < 4096 {
		return nil, fmt.Errorf("pbsgpu: index image too short")
	}
	var cr *C.pbsgpu_crypt
	if c != nil {
		cr = c.c
	}
	var r *C.pbsgpu_reader
	if err := e.err(C.pbsgpu_reader_open_fidx(e.ctx, (*C.uint8_t)(unsafe.Pointer(&fidx[0])), C.uint64_t(len(fidx)), cr,
		C.uint64_t(cacheBytes), &r)); err != nil {
		return nil, err
	}
	dg := make([][32]byte, (len(fidx)-4096)/32)
	for i := range dg {
		copy(dg[i][:], fidx[4096+32*i:4096+32*i+32])
	}
	return &PayloadReader{e: e, r: r, source: source, digests: dg, size: uint64(C.pbsgpu_reader_size(r))}, nil
}

// RestoreImage writes the whole image of an image reader (NewImageReader) to f, sparsely
// (pbsgpu_reader_read_sparse): per slice of sliceBytes (0 = 1 GiB), one plan that leaves out the zero chunks, one fetch
// of the named blobs, one read that returns only the data extents, and a WriteAt of each; then f.Truncate to the image's
// size.  Zero chunks are never fetched or decoded and no all-zero 4 KiB block is written, so f must read as zeros where
// nothing is written: a new file (which stays thin) or a device the caller zeroed, as upstream's skip-zero restore.
func (p *PayloadReader) RestoreImage(f *os.File, sliceBytes uint64) error {
	if sliceBytes == 0 {
		sliceBytes = 1 << 30
	}
	if sliceBytes > p.size {
		sliceBytes = p.size
	}
	out := make([]byte, sliceBytes+1) // the packed data of one slice, reused by every slice (+1: never empty)
	for off := uint64(0); off < p.size; off += sliceBytes {
		n := p.size - off
		if n > sliceBytes {
			n = sliceBytes
		}
		o, l := []uint64{off}, []uint64{n}
		blobs, bo, bl, need, err := p.fetch(o, l, C.PBSGPU_READ_SPARSE)
		if err != nil {
			return err
		}
		parts := (off+n-1)/4096 - off/4096 + 1
		extCap := (parts + 1) / 2
		ext := make([]uint64, 2*extCap)
		extFirst := make([]uint64, 2)
		outOff := []uint64{0}
		status := make([]int32, 1)
		blobStatus := make([]int32, len(need))
		rc := C.pbsgpu_reader_read_sparse(p.r, (*C.uint64_t)(unsafe.Pointer(&o[0])), (*C.uint64_t)(unsafe.Pointer(&l[0])), 1, 0,
			unsafe.Pointer(&blobs[0]), (*C.uint64_t)(unsafe.Pointer(&bo[0])), (*C.uint64_t)(unsafe.Pointer(&bl[0])),
			(*C.uint64_t)(unsafe.Pointer(&need[0])), C.uint32_t(len(need)-1), (*C.uint8_t)(unsafe.Pointer(&out[0])),
			(*C.uint64_t)(unsafe.Pointer(&outOff[0])), (*C.uint64_t)(unsafe.Pointer(&ext[0])), C.uint64_t(extCap),
			(*C.uint64_t)(unsafe.Pointer(&extFirst[0])), (*C.int32_t)(unsafe.Pointer(&status[0])),
			(*C.int32_t)(unsafe.Pointer(&blobStatus[0])))
		if err := p.e.err(rc); err != nil {
			return err
		}
		if status[0] != int32(C.PBSGPU_DEC_OK) {
			for j, s := range blobStatus[:len(need)-1] {
				if s != int32(C.PBSGPU_DEC_OK) {
					return fmt.Errorf("pbsgpu: image chunk %d (%x): status %d", need[j], p.digests[need[j]], s)
				}
			}
			return fmt.Errorf("pbsgpu: image slice at %d: status %d", off, status[0])
		}
		var at uint64
		for e := extFirst[0]; e < extFirst[1]; e++ {
			eo, el := ext[2*e], ext[2*e+1]
			if _, err := f.WriteAt(out[at:at+el], int64(eo)); err != nil {
				return err
			}
			at += el
		}
	}
	return f.Truncate(int64(p.size))
}

// RestoreFile is one regular file of RestoreFiles: where it goes, st_mode, mtime in seconds, the payload offset of its
// PAYLOAD header and its size.
type RestoreFile struct {
	Path          string
	Mode          uint32
	Mtime         int64
	PayloadOffset uint64
	Size          uint64
}

// readFileSparse reads ranges of files sparsely (pbsgpu_reader_plan_file_sparse, _read_file_sparse): range i is the
// content bytes [pos[i], pos[i] + n[i]) of file fs[i].  It returns per range its (content offset, length) extents and
// its packed data bytes, which are slices of out (grown only when it is too small; RestoreFiles sizes it once).
func (p *PayloadReader) readFileSparse(fs []*RestoreFile, pos, n []uint64, out []byte) ([][][2]uint64, [][]byte, error) {
	k := len(fs)
	fo, sz := make([]uint64, k), make([]uint64, k)
	outOff := make([]uint64, k)
	var total, extCap uint64
	for i, f := range fs {
		fo[i], sz[i], outOff[i] = f.PayloadOffset, f.Size, total
		total += n[i]
		if n[i] > 0 {
			extCap += ((pos[i]+n[i]-1)/4096 - pos[i]/4096 + 2) / 2
		}
	}
	need := make([]uint64, len(p.digests)+1)
	var nk C.uint64_t
	if err := p.e.err(C.pbsgpu_reader_plan_file_sparse(p.r, (*C.uint64_t)(unsafe.Pointer(&fo[0])),
		(*C.uint64_t)(unsafe.Pointer(&sz[0])), (*C.uint64_t)(unsafe.Pointer(&pos[0])), (*C.uint64_t)(unsafe.Pointer(&n[0])),
		C.uint32_t(k), (*C.uint64_t)(unsafe.Pointer(&need[0])), nil, C.uint64_t(len(need)), &nk)); err != nil {
		return nil, nil, err
	}
	need = need[:nk]
	var blobs []byte
	bo, bl := make([]uint64, nk+1), make([]uint64, nk+1)
	for j, c := range need {
		b, err := p.source(p.digests[c])
		if err != nil {
			return nil, nil, err
		}
		bo[j], bl[j] = uint64(len(blobs)), uint64(len(b))
		blobs = append(blobs, b...)
	}
	blobs, need = append(blobs, 0), append(need, 0)
	if uint64(len(out)) < total+1 {
		out = make([]byte, total+1)
	}
	ext := make([]uint64, 2*extCap+2)
	extFirst := make([]uint64, k+1)
	status := make([]int32, k)
	rc := C.pbsgpu_reader_read_file_sparse(p.r, (*C.uint64_t)(unsafe.Pointer(&fo[0])), (*C.uint64_t)(unsafe.Pointer(&sz[0])),
		(*C.uint64_t)(unsafe.Pointer(&pos[0])), (*C.uint64_t)(unsafe.Pointer(&n[0])), C.uint32_t(k), unsafe.Pointer(&blobs[0]),
		(*C.uint64_t)(unsafe.Pointer(&bo[0])), (*C.uint64_t)(unsafe.Pointer(&bl[0])), (*C.uint64_t)(unsafe.Pointer(&need[0])),
		C.uint32_t(len(need)-1), (*C.uint8_t)(unsafe.Pointer(&out[0])), (*C.uint64_t)(unsafe.Pointer(&outOff[0])),
		(*C.uint64_t)(unsafe.Pointer(&ext[0])), C.uint64_t(extCap), (*C.uint64_t)(unsafe.Pointer(&extFirst[0])),
		(*C.int32_t)(unsafe.Pointer(&status[0])), nil)
	if err := p.e.err(rc); err != nil {
		return nil, nil, err
	}
	exts, packed := make([][][2]uint64, k), make([][]byte, k)
	for i, f := range fs {
		if status[i] != int32(C.PBSGPU_DEC_OK) {
			return nil, nil, fmt.Errorf("pbsgpu: restore of %s (payload offset %d, %d bytes): status %d", f.Path,
				f.PayloadOffset, f.Size, status[i])
		}
		at := outOff[i]
		for e := extFirst[i]; e < extFirst[i+1]; e++ {
			exts[i] = append(exts[i], [2]uint64{ext[2*e], ext[2*e+1]})
		}
		var m uint64
		for _, x := range exts[i] {
			m += x[1]
		}
		packed[i] = out[at : at+m]
	}
	return exts, packed, nil
}

// writeExtents writes the packed bytes of a file's extents at their content offsets.
func writeExtents(f *os.File, exts [][2]uint64, packed []byte) error {
	var at uint64
	for _, x := range exts {
		if _, err := f.WriteAt(packed[at:at+x[1]], int64(x[0])); err != nil {
			return err
		}
		at += x[1]
	}
	return nil
}

// RestoreFiles writes files of a payload reader into place sparsely (the replacement for restoreFile's io.Copy,
// internal/pxar/restore.go): zero chunks are never fetched or decoded, and each file gets one WriteAt per data extent
// (4 KiB blocks aligned to its content start that are not all zero) and a Truncate to its size, so its zero blocks stay
// holes.  Files up to sliceBytes (0 = 1 GiB) go in batches of about sliceBytes file bytes, one read per batch; a larger
// file is read in pieces of sliceBytes rounded down to a multiple of 4096.  A file whose size matches, and its mtime
// too unless noAttr, is not rewritten unless it is a directory or a symlink (shouldUpdateFile, as the Python mirror).
// One output buffer of sliceBytes serves every read.  Unless noAttr, each file gets its mode's permission bits and
// mtime.  Directories and symlinks are the caller's (they need no archive bytes).
func (p *PayloadReader) RestoreFiles(files []RestoreFile, noAttr bool, sliceBytes uint64) error {
	if sliceBytes == 0 {
		sliceBytes = 1 << 30
	}
	piece := sliceBytes / 4096 * 4096
	if piece == 0 {
		piece = 4096
	}
	create := func(f *RestoreFile) (*os.File, error) {
		return os.OpenFile(f.Path, os.O_CREATE|os.O_TRUNC|os.O_WRONLY, 0666)
	}
	finish := func(w *os.File, f *RestoreFile) error {
		err := w.Truncate(int64(f.Size))
		if cerr := w.Close(); err == nil {
			err = cerr
		}
		if err != nil || noAttr {
			return err
		}
		if err := os.Chmod(f.Path, os.FileMode(f.Mode&0777)); err != nil {
			return err
		}
		t := time.Unix(f.Mtime, 0)
		return os.Chtimes(f.Path, t, t)
	}
	out := make([]byte, piece+1) // the packed data of one batch or piece, reused by every read
	var batch []*RestoreFile
	var acc uint64
	flush := func() error {
		if len(batch) == 0 {
			return nil
		}
		pos, n := make([]uint64, len(batch)), make([]uint64, len(batch))
		for i, f := range batch {
			n[i] = f.Size
		}
		exts, packed, err := p.readFileSparse(batch, pos, n, out)
		if err != nil {
			return err
		}
		for i, f := range batch {
			w, err := create(f)
			if err != nil {
				return err
			}
			if err := writeExtents(w, exts[i], packed[i]); err != nil {
				w.Close()
				return err
			}
			if err := finish(w, f); err != nil {
				return err
			}
		}
		batch, acc = batch[:0], 0
		return nil
	}
	for i := range files {
		f := &files[i]
		// shouldUpdateFile: keep what is there unless it is a directory or a symlink, or its size (or, unless noAttr,
		// its mtime) differs
		if st, err := os.Lstat(f.Path); err == nil && !st.IsDir() && st.Mode()&os.ModeSymlink == 0 &&
			uint64(st.Size()) == f.Size && (noAttr || st.ModTime().Unix() == f.Mtime) {
			if !noAttr {
				if err := os.Chmod(f.Path, os.FileMode(f.Mode&0777)); err != nil {
					return err
				}
				t := time.Unix(f.Mtime, 0)
				if err := os.Chtimes(f.Path, t, t); err != nil {
					return err
				}
			}
			continue
		}
		if f.Size > piece {
			if err := flush(); err != nil {
				return err
			}
			w, err := create(f)
			if err != nil {
				return err
			}
			for lo := uint64(0); lo < f.Size; lo += piece {
				m := min(piece, f.Size-lo)
				exts, packed, err := p.readFileSparse([]*RestoreFile{f}, []uint64{lo}, []uint64{m}, out)
				if err == nil {
					err = writeExtents(w, exts[0], packed[0])
				}
				if err != nil {
					w.Close()
					return err
				}
			}
			if err := finish(w, f); err != nil {
				return err
			}
			continue
		}
		if len(batch) > 0 && acc+f.Size > piece {
			if err := flush(); err != nil {
				return err
			}
		}
		batch = append(batch, f)
		acc += f.Size
	}
	return flush()
}

// ZipWriter writes one <name>.zip of a restore (the replacement for zip.NewWriter + io.Copy(rangeReader) in
// createZipForSource, internal/pxar/zip.go): files are deflated on the GPU from a PayloadReader
// (pbsgpu_reader_read_deflate) and the container is written by pbsgpu_zip_*.  Every entry but a directory has flag bit
// 3 and a data descriptor; Close writes the central directory.  Files up to PieceBytes go in batches of about PieceBytes
// file bytes, one read per batch; a larger file goes in 128 KiB-aligned pieces of plain ranges continued with `more`,
// after one plain read of its 16-byte PAYLOAD header, and its CRC-32 is combined from the pieces'.  LZC: deflate with
// the hash-chain parse (pbsgpu_deflate_batch_lzc), for a smaller zip at a lower rate; false writes the greedy parse's.
type ZipWriter struct {
	pr         *PayloadReader
	w          io.Writer
	PieceBytes uint64
	LZC        bool
	pos        uint64
	entries    []C.pbsgpu_zip_entry
}

// ZipFile is one regular file of AddFiles: its path in the archive, st_mode, mtime and place in the payload stream.
type ZipFile struct {
	Path          string
	Mode          uint32
	Mtime         int64
	PayloadOffset uint64
	Size          uint64
}

func (e *Engine) NewZipWriter(pr *PayloadReader, w io.Writer) *ZipWriter {
	return &ZipWriter{pr: pr, w: w, PieceBytes: 1 << 30}
}

func (z *ZipWriter) write(b []byte) error {
	_, err := z.w.Write(b)
	z.pos += uint64(len(b))
	return err
}

func zipRecord(f func(out *C.uint8_t, cap C.uint64_t) C.uint64_t) []byte {
	need := uint64(f(nil, 0))
	out := make([]byte, need+1)
	f((*C.uint8_t)(unsafe.Pointer(&out[0])), C.uint64_t(need))
	return out[:need]
}

func (z *ZipWriter) entry(name string, mode uint32, mtime int64, method uint32, size uint64) *C.pbsgpu_zip_entry {
	e := C.pbsgpu_zip_entry{name: (*C.uint8_t)(C.CBytes([]byte(name + "\x00"))), name_len: C.uint32_t(len(name)), mode: C.uint32_t(mode),
		mtime: C.int64_t(mtime), method: C.uint32_t(method), size: C.uint64_t(size), offset: C.uint64_t(z.pos)}
	z.entries = append(z.entries, e)
	return &z.entries[len(z.entries)-1]
}

func (z *ZipWriter) localHeader(e *C.pbsgpu_zip_entry) error {
	return z.write(zipRecord(func(o *C.uint8_t, c C.uint64_t) C.uint64_t { return C.pbsgpu_zip_local_header(e, o, c) }))
}

func (z *ZipWriter) descriptor(e *C.pbsgpu_zip_entry) error {
	return z.write(zipRecord(func(o *C.uint8_t, c C.uint64_t) C.uint64_t { return C.pbsgpu_zip_data_descriptor(e, o, c) }))
}

// AddDirectory adds a directory entry (its name gets a trailing '/').
func (z *ZipWriter) AddDirectory(path string, mode uint32, mtime int64) error {
	if !strings.HasSuffix(path, "/") {
		path += "/"
	}
	return z.localHeader(z.entry(path, mode, mtime, 0, 0))
}

// AddSymlink adds a symlink entry: stored, the target as content.
func (z *ZipWriter) AddSymlink(path, target string, mode uint32, mtime int64) error {
	e := z.entry(path, mode, mtime, 0, uint64(len(target)))
	e.crc, e.comp_size = C.uint32_t(crc32.ChecksumIEEE([]byte(target))), C.uint64_t(len(target))
	if err := z.localHeader(e); err != nil {
		return err
	}
	if err := z.write([]byte(target)); err != nil {
		return err
	}
	return z.descriptor(e)
}

// AddFiles adds regular files, deflated on the GPU.
func (z *ZipWriter) AddFiles(files []ZipFile) error {
	piece := z.PieceBytes / (128 << 10) * (128 << 10)
	if piece == 0 {
		piece = 128 << 10
	}
	var batch []ZipFile
	var acc uint64
	flush := func() error {
		if len(batch) == 0 {
			return nil
		}
		off, size := make([]uint64, len(batch)), make([]uint64, len(batch))
		for i, f := range batch {
			off[i], size[i] = f.PayloadOffset, f.Size
		}
		streams, crcs, err := z.pr.readDeflate(off, size, true, nil, z.LZC)
		if err != nil {
			return err
		}
		for i, f := range batch {
			e := z.entry(f.Path, f.Mode, f.Mtime, 8, f.Size)
			e.crc, e.comp_size = C.uint32_t(crcs[i]), C.uint64_t(len(streams[i]))
			if err := z.localHeader(e); err != nil {
				return err
			}
			if err := z.write(streams[i]); err != nil {
				return err
			}
			if err := z.descriptor(e); err != nil {
				return err
			}
		}
		batch, acc = batch[:0], 0
		return nil
	}
	for _, f := range files {
		if f.Size > piece {
			if err := flush(); err != nil {
				return err
			}
			if err := z.large(f, piece); err != nil {
				return err
			}
			continue
		}
		if len(batch) > 0 && acc+f.Size > piece {
			if err := flush(); err != nil {
				return err
			}
		}
		batch = append(batch, f)
		acc += f.Size
	}
	return flush()
}

func (z *ZipWriter) large(f ZipFile, piece uint64) error {
	hdr := make([]byte, 16)
	if err := z.pr.read([]uint64{f.PayloadOffset}, []uint64{16}, false, hdr, []uint64{0}); err != nil {
		return err
	}
	if !bytes.Equal(hdr, header(pxarPayload, 16+f.Size)) {
		return fmt.Errorf("pbsgpu: file at payload offset %d (%d bytes): bad PAYLOAD header", f.PayloadOffset, f.Size)
	}
	e := z.entry(f.Path, f.Mode, f.Mtime, 8, f.Size)
	if err := z.localHeader(e); err != nil {
		return err
	}
	var crc uint32
	var csize uint64
	for lo := uint64(0); lo < f.Size; {
		n := f.Size - lo
		if n > piece {
			n = piece
		}
		more := []uint8{0}
		if lo+n < f.Size {
			more[0] = 1
		}
		s, c, err := z.pr.readDeflate([]uint64{f.PayloadOffset + 16 + lo}, []uint64{n}, false, more, z.LZC)
		if err != nil {
			return err
		}
		crc = uint32(C.pbsgpu_crc32_combine(C.uint32_t(crc), C.uint32_t(c[0]), C.uint64_t(n)))
		csize += uint64(len(s[0]))
		if err := z.write(s[0]); err != nil {
			return err
		}
		lo += n
	}
	e.crc, e.comp_size = C.uint32_t(crc), C.uint64_t(csize)
	return z.descriptor(e)
}

// Close writes the central directory and its end records, and frees the names.
func (z *ZipWriter) Close() error {
	var ep *C.pbsgpu_zip_entry
	if len(z.entries) > 0 {
		ep = &z.entries[0]
	}
	n := C.uint64_t(len(z.entries))
	err := z.write(zipRecord(func(o *C.uint8_t, c C.uint64_t) C.uint64_t { return C.pbsgpu_zip_directory(ep, n, C.uint64_t(z.pos), o, c) }))
	for i := range z.entries {
		C.free(unsafe.Pointer(z.entries[i].name))
	}
	z.entries = nil
	return err
}
