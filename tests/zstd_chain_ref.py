"""Restatement of the compressed DataBlob format with a hash-chain match search over the whole chunk and a lazy parse
(pbsgpu_blob_encode_batch_lzc, K16 in csrc/zchain.cu plus K9b / K10) in numpy / pure Python.  Test infrastructure: the
GPU output is compared with it byte for byte, and libzstd's decoder checks it (tests/test_zstd_chain_cpu.py).  The
sequences section and the literals are tests/zstd_huf_ref.py's block_content_lzh, unchanged.

The frame is _lzh's (single segment, 128 KiB blocks, a constant block is an RLE_Block, a block stays raw unless its
content is strictly smaller); only the sequences of a block that is not constant change:
  prev(i)   for i <= len - CH_MINMATCH: the largest j < i of the same chunk whose CH_MINMATCH bytes equal i's (exact
            byte equality, so every chain step is a real match and prev does not depend on any order of work).
  best(i)   among the first CH_DEPTH chain entries j = prev(i), prev(prev(i)), ... with i - j <= CH_MAXDIST, the
            longest match, extended forward to the end of i's block and no further; ties go to the nearer entry.  The
            source may lie in any earlier block of the chunk (constant blocks too) and may overlap i.  A position with
            fewer than CH_MINMATCH bytes left in its block has no match.
  parse     per block from its first position: at a match m, while best(m + 1) exists and its gain is larger than
            best(m)'s by more than CH_MARGIN, m becomes a literal and the parse moves on (at most CH_LAZY times);
            gain = 4 L - floor(log2(offset + 3)).  Then (literal run, length, offset) is emitted and the parse jumps
            past the match.  No repeat offsets: every block decodes against the decoded window alone.
The constants define the output bytes; csrc/zchain.cuh holds the same values, DESIGN.md K16 the table they come from."""
from __future__ import annotations

from array import array

import numpy as np

from oracle.pyref import BLOB_MAGIC_COMPRESSED, BLOB_MAGIC_UNCOMPRESSED, ZFRAME_BLOCK
from zstd_huf_ref import block_content_lzh

CH_MINMATCH = 4              # chain key: 4 bytes, the shortest match
CH_DEPTH = 16                # chain entries searched per position
CH_LAZY = 2                  # positions the parse may move on from a match
CH_MARGIN = 4                # gain a later match must exceed the current one's by
CH_MAXDIST = (1 << 24) - 4   # the largest offset: K9's packed sequences keep it in 24 bits


def chains(a: np.ndarray, minmatch: int = CH_MINMATCH) -> np.ndarray:
    """prev(i) for i <= len - minmatch (-1: none); the array has max(0, len - minmatch + 1) entries."""
    n = len(a) - minmatch + 1
    if n <= 0:
        return np.zeros(0, np.int64)
    b = a.astype(np.uint64)
    key = np.zeros(n, np.uint64)
    for k in range(minmatch):
        key |= b[k:k + n] << np.uint64(8 * k)
    order = np.argsort(key, kind="stable")
    prev = np.full(n, -1, np.int64)
    same = key[order[1:]] == key[order[:-1]]
    prev[order[1:][same]] = order[:-1][same]
    return prev


def _mlen(d: bytes, i: int, j: int, lim: int) -> int:
    """The common length of d[i:lim] and d[j:], j < i (the source may overlap)."""
    L, step = 0, 16
    while i + L < lim:
        n = min(step, lim - i - L)
        if d[j + L:j + L + n] == d[i + L:i + L + n]:
            L += n
            step *= 2
            continue
        while n > 1:   # the first difference lies in [L, L + n)
            h = n // 2
            if d[j + L:j + L + h] == d[i + L:i + L + h]:
                L += h
                n -= h
            else:
                n = h
        return L
    return L


class _Search:
    """best(i) of one chunk, computed on demand."""

    def __init__(self, d: bytes, depth: int, minmatch: int, maxdist: int):
        self.d, self.depth, self.minmatch, self.maxdist = d, depth, minmatch, maxdist
        self.prev = array("q", chains(np.frombuffer(d, np.uint8), minmatch).tobytes())

    def best(self, i: int, lim: int):
        """(length, offset) of best(i) in the block that ends at lim; (0, 0) for none."""
        if i + self.minmatch > lim:
            return 0, 0
        j, k, bl, bo = self.prev[i], 0, 0, 0
        while j >= 0 and k < self.depth and i - j <= self.maxdist:
            L = _mlen(self.d, i, j, lim)
            if L > bl:
                bl, bo = L, i - j
                if L == lim - i:
                    break
            j, k = self.prev[j], k + 1
        return (bl, bo) if bl >= self.minmatch else (0, 0)


def gain(L: int, off: int) -> int:
    return 4 * L - ((off + 3).bit_length() - 1)


def chain_parse(s: _Search, start: int, lim: int, lazy: int = CH_LAZY, margin: int = CH_MARGIN):
    """The parse of block [start, lim) of the chunk -> (literals, sequences (literal run, length, offset))."""
    d = s.d
    lits, seqs = [], []
    run = i = start
    while i + s.minmatch <= lim:
        L, o = s.best(i, lim)
        if not L:
            i += 1
            continue
        for _ in range(lazy):
            L2, o2 = s.best(i + 1, lim)
            if not L2 or gain(L2, o2) <= gain(L, o) + margin:
                break
            i, L, o = i + 1, L2, o2
        lits.append(d[run:i])
        seqs.append((i - run, L, o))
        i = run = i + L
    lits.append(d[run:lim])
    return b"".join(lits), seqs


def zstd_frame_lzc(data: bytes, depth: int = CH_DEPTH, lazy: int = CH_LAZY, margin: int = CH_MARGIN,
                   minmatch: int = CH_MINMATCH) -> bytes:
    """zstd_huf_ref.zstd_frame_lzh's frame with chain_parse as the parse of every block that is not constant."""
    data = bytes(data)
    out = bytearray(b"\x28\xb5\x2f\xfd\xe0" + len(data).to_bytes(8, "little"))
    nb = max(1, (len(data) + ZFRAME_BLOCK - 1) // ZFRAME_BLOCK)
    s = _Search(data, depth, minmatch, CH_MAXDIST)
    for b in range(nb):
        lo, hi = b * ZFRAME_BLOCK, min(len(data), (b + 1) * ZFRAME_BLOCK)
        blk = data[lo:hi]
        last = int(b + 1 == nb)
        if len(blk) > 0 and blk.count(blk[:1]) == len(blk):
            out += (last | 1 << 1 | len(blk) << 3).to_bytes(3, "little") + blk[:1]
            continue
        body = block_content_lzh(*chain_parse(s, lo, hi, lazy, margin)) if blk else blk
        if len(body) < len(blk):
            out += (last | 2 << 1 | len(body) << 3).to_bytes(3, "little") + body
        else:
            out += (last | len(blk) << 3).to_bytes(3, "little") + blk
    return bytes(out)


def blob_encode_lzc(data: bytes) -> bytes:
    """blob_encode with zstd_frame_lzc as the compressed payload (kept only when smaller than the raw bytes)."""
    import zlib
    data = bytes(data)
    if data:
        fr = zstd_frame_lzc(data)
        if len(fr) < len(data):
            return BLOB_MAGIC_COMPRESSED + zlib.crc32(fr).to_bytes(4, "little") + fr
    return BLOB_MAGIC_UNCOMPRESSED + zlib.crc32(data).to_bytes(4, "little") + data


# -- test data ---------------------------------------------------------------------------------------------------------
def half_zero(nbytes: int, seed: int = 0, run: int = 4096) -> np.ndarray:
    """Random bytes in which about half of the `run`-byte stretches are zeros."""
    rng = np.random.default_rng(seed)
    out = rng.integers(0, 256, nbytes, dtype=np.uint8)
    for k in np.flatnonzero(rng.random((nbytes + run - 1) // run) < 0.5):
        out[k * run:(k + 1) * run] = 0
    return out
