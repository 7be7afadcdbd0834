"""Restatement of the sparse image restore's output (include/pbsgpu.h, pbsgpu_reader_read_sparse) in pure Python.  Test
infrastructure: the GPU's extents and packed bytes are compared against it.

- Image offsets are cut into 4096-byte blocks aligned to the image: block b is [4096 b, 4096 (b + 1)).
- Within a range, a block's part inside the range is a hole when all of its bytes are zero.
- The data extents of the range are the maximal runs of non-hole block parts, as (image offset, length), ascending; the
  packed output is their bytes, concatenated in that order.
- A range of B block parts has at most ceil(B / 2) extents (every other part a hole).
- Zero chunk: a chunk whose index digest is the digest of as many zero bytes (plain, or keyed SHA-256(zeros || id_key)).
  It is served by its digest when its bounds are block boundaries (served_by_digest); the extents do not depend on it.
"""
from __future__ import annotations

import hashlib

BLOCK = 4096


def block_parts(off: int, length: int) -> list[tuple[int, int]]:
    """The [lo, hi) block parts of the range [off, off + length), ascending."""
    out, a, end = [], off, off + length
    while a < end:
        hi = min(end, (a // BLOCK + 1) * BLOCK)
        out.append((a, hi))
        a = hi
    return out


def extents(image: bytes, off: int, length: int) -> list[tuple[int, int]]:
    """The data extents of the range: maximal runs of block parts with a non-zero byte."""
    out: list[tuple[int, int]] = []
    for lo, hi in block_parts(off, length):
        if image[lo:hi].count(0) != hi - lo:
            if out and out[-1][0] + out[-1][1] == lo:
                out[-1] = (out[-1][0], out[-1][1] + hi - lo)
            else:
                out.append((lo, hi - lo))
    return out


def packed(image: bytes, ext: list[tuple[int, int]]) -> bytes:
    return b"".join(image[a:a + n] for a, n in ext)


def ext_bound(off: int, length: int) -> int:
    """ceil(B / 2) for the B block parts of the range: the most extents it can have."""
    return (len(block_parts(off, length)) + 1) // 2


def zero_digest(n: int, id_key: bytes | None = None) -> bytes:
    """The index digest of a chunk of n zero bytes: SHA-256, or keyed SHA-256(zeros || id_key)."""
    return hashlib.sha256(b"\0" * n + (id_key or b"")).digest()


def served_by_digest(start: int, end: int, size: int) -> bool:
    """A zero chunk [start, end) of an image of `size` bytes is served by its digest when both bounds are block
    boundaries (the end may be the image's end); any other zero chunk shares a block with its neighbours and is read
    like a data chunk."""
    return start % BLOCK == 0 and (end % BLOCK == 0 or end == size)


def holes(image: bytes, size: int) -> list[tuple[int, int]]:
    """The whole 4 KiB-aligned blocks of the image that are all zero, merged into [lo, hi) runs (the last, short block
    counts when it is all zero)."""
    out: list[tuple[int, int]] = []
    for lo, hi in block_parts(0, size):
        if image[lo:hi].count(0) == hi - lo:
            if out and out[-1][1] == lo:
                out[-1] = (out[-1][0], hi)
            else:
                out.append((lo, hi))
    return out
