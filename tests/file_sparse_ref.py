"""Restatement of the sparse file restore's output (include/pbsgpu.h, pbsgpu_reader_read_file_sparse) in pure Python.
Test infrastructure: the GPU's extents and packed bytes are compared against it.

- A range is the content bytes [pos, pos + len) of one file.  Content offsets are cut into 4096-byte blocks aligned to
  the file's content start: block b is content bytes [4096 b, 4096 (b + 1)).
- Within the range, a block's part is a hole when all of its bytes are zero; the extents are the maximal runs of the
  other parts as (content offset, length), ascending, and the packed output is their bytes in that order.  This is the
  image form of tests/sparse_ref.py applied to the file's content, so a range of B block parts has at most ceil(B / 2)
  extents.
- Zero chunk of a .didx index: a chunk whose length is the index's longest and whose digest is the digest of that many
  zero bytes (plain, or keyed SHA-256(zeros || id_key)), when two or more chunks of that length share a digest;
  otherwise there are none (the zero digest is not computed for a digest the index holds once).  The 64-byte buzhash
  window of zero bytes is XOR_{j<64} rotl(T[0], j mod 32): every rotation occurs twice, so it is 0 under any table and
  never a candidate
  (the threshold mask - 2 is above 0).  A zero run is therefore cut only at the chunker's maximum (or where a file start
  is suggested), and that one length carries almost all zero chunks.
"""
from __future__ import annotations

import numpy as np

import scan_ref
import sparse_ref

BLOCK = sparse_ref.BLOCK
PAYLOAD = 0x28147A1B0B7C1A25
START_MARKER = 0x834C68C2194A4ED2
TAIL_MARKER = 0x6C72B78B984C81B5


def extents(content: bytes, pos: int, length: int) -> list[tuple[int, int]]:
    """The data extents of the content range [pos, pos + length), in content offsets."""
    return sparse_ref.extents(content, pos, length)


def packed(content: bytes, ext: list[tuple[int, int]]) -> bytes:
    return sparse_ref.packed(content, ext)


def ext_bound(pos: int, length: int) -> int:
    return sparse_ref.ext_bound(pos, length)


def zero_window_hash(table) -> int:
    """The buzhash of a 64-byte window of zero bytes under `table`, written out as the XOR of its rotations."""
    t0, h = int(table[0]) & 0xFFFFFFFF, 0
    for j in range(scan_ref.WINDOW):
        r = j % 32
        h ^= ((t0 << r) | (t0 >> (32 - r))) & 0xFFFFFFFF if r else t0
    return h


def zero_chunks(ends, digests, id_key: bytes | None = None) -> set[int]:
    """The chunks of an index (end offsets, 32-byte digests) that the rule serves by digest."""
    ends = [int(e) for e in ends]
    lens = [e - (ends[k - 1] if k else 0) for k, e in enumerate(ends)]
    if not lens:
        return set()
    longest = max(lens)
    seen = [bytes(digests[k]) for k, n in enumerate(lens) if n == longest]
    if len(set(seen)) == len(seen):
        return set()
    z = sparse_ref.zero_digest(longest, id_key)
    return {k for k, n in enumerate(lens) if n == longest and bytes(digests[k]) == z}


def payload_header(size: int) -> bytes:
    return PAYLOAD.to_bytes(8, "little") + (16 + size).to_bytes(8, "little")


def payload_stream(files: list[bytes]) -> tuple[bytes, list[int]]:
    """The pxar v2 payload stream transfer.PayloadStreamWriter writes for these files -> (stream, payload offsets)."""
    parts, offs, at = [START_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little")], [], 16
    for f in files:
        offs.append(at)
        parts.append(payload_header(len(f)) + f)
        at += 16 + len(f)
    parts.append(TAIL_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little"))
    return b"".join(parts), offs


def stream_ends(cfg, stream: bytes, offs: list[int]) -> list[int]:
    """The chunk ends of the stream as the payload chunker cuts it: the buzhash candidates, the min/max rule and a
    suggested boundary at every file's header (tests/scan_ref.py)."""
    table = np.array(list(cfg.table), dtype=np.uint32)
    cands = scan_ref.candidates(table, int(cfg.mask), stream)
    return scan_ref.resolve(cands, len(stream), cfg, forced=offs)
