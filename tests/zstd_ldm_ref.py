"""Restatement of the compressed DataBlob format with long-distance matches (pbsgpu_blob_encode_batch_lzl, K12 in
csrc/zldm.cu plus K9 / K10 with long spans) in numpy / pure Python.  Test infrastructure: the GPU output is compared
with it byte for byte, and libzstd's decoder checks it (tests/test_zstd_ldm_cpu.py).  The block parse, the sequences
section and the literals are tests/zstd_lz_ref.py's, tests/zstd_ent_ref.py's and tests/zstd_huf_ref.py's, unchanged.

_lzl is _lzh plus long matches that reach anywhere earlier in the same chunk (the frame is single-segment, so its
window is the whole chunk):
  anchors    a 64-bit gear hash over the 64 bytes ending at i, h = (h << 1) + G[byte] (a byte leaves it after 64
             shifts); i is an anchor when the top LDM_RATE bits of h are zero, and h is its fingerprint.  Only positions
             with a full window in the chunk (i >= 63) count.
  candidates cand(a): the latest earlier anchor with a's fingerprint, if a - cand(a) <= LDM_MAXDIST and the two 64-byte
             windows are equal (nothing older is searched).  The match [s, e) at offset d = a - cand(a) is the window
             extended backward while s - 1 >= d (neither side goes below the chunk start) and forward to the chunk end,
             as long as the bytes at x and x - d are equal.  The source may overlap the destination.
  selection  the matches sorted by (s, e descending, d); cur = 0; per match s' = max(s, cur); [s', e) is kept when
             e - s' >= LDM_MINMATCH, and then cur = e.  A kept match is split at the 128 KiB block edges; pieces in
             constant blocks (RLE_Blocks) and pieces shorter than LZ_MINMATCH are dropped.  The rest are the block's
             long spans.
  block      lz_parse with the spans: K9's candidates unchanged; a span is taken where it starts and the parse jumps
             past it; a short match is cut at the next span's start and kept only while it is still >= LZ_MINMATCH
             long (else its first byte is a literal).  The block's content is the smaller of its _lzh content and
             this parse's (block_content_lzh of both), _lzh on ties; no repeat offsets, so every block decodes on its
             own against the decoded window.  A block without spans is _lzh's, and every _lzl blob is at most its _lzh
             blob.
The constants define the output bytes; csrc/zldm.cuh holds the same values, DESIGN.md K12 the sweep LDM_RATE is from."""
from __future__ import annotations

import numpy as np

from oracle.pyref import BLOB_MAGIC_COMPRESSED, BLOB_MAGIC_UNCOMPRESSED, ZFRAME_BLOCK
from zstd_huf_ref import block_content_lzh
from zstd_lz_ref import LZ_HBITS, LZ_MINMATCH, LZ_TILE, lz_candidates, lz_parse

LDM_RATE = 7                   # an anchor where the top 7 bits of the hash are zero: about one per 128 bytes
LDM_WINDOW = 64                # bytes hashed per anchor
LDM_MINMATCH = 64              # shortest kept long match
LDM_MAXDIST = (1 << 24) - 4    # the largest offset: K9's sequences keep it in 24 bits
LDM_SEED = 0                   # splitmix64 seed of the gear table: the first for which no run of one byte value has an
                               # anchor, so constant runs add none
_M64 = (1 << 64) - 1


def gear_table(seed: int = LDM_SEED) -> np.ndarray:
    """256 values of splitmix64 from `seed`."""
    out, x = [], seed
    for _ in range(256):
        x = (x + 0x9E3779B97F4A7C15) & _M64
        z = x
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
        out.append(z ^ (z >> 31))
    return np.array(out, np.uint64)


GEAR = gear_table()


def gear_hashes(a: np.ndarray) -> np.ndarray:
    """h(i) for every i; only i >= 63 are window hashes.  Doubling: h_2k(i) = (h_k(i - k) << k) + h_k(i)."""
    with np.errstate(over="ignore"):
        h = GEAR[a]
        k = 1
        while k < LDM_WINDOW:
            h2 = h.copy()
            h2[k:] = (h[:-k] << np.uint64(k)) + h[k:]
            h, k = h2, 2 * k
    return h


def anchors(a: np.ndarray, rate: int = LDM_RATE):
    """(positions, fingerprints) of the anchors of a chunk, in position order."""
    if len(a) < LDM_WINDOW:
        return np.zeros(0, np.int64), np.zeros(0, np.uint64)
    h = gear_hashes(a)[LDM_WINDOW - 1:]
    pos = np.flatnonzero((h >> np.uint64(64 - rate)) == 0)
    return pos + LDM_WINDOW - 1, h[pos]


def _run_back(a: np.ndarray, x: int, lo: int, d: int) -> int:
    """The smallest s in [lo, x] with a[y] == a[y - d] for all y in [s, x)."""
    while x > lo:
        k = max(lo, x - 4096)
        ne = np.flatnonzero(a[k:x] != a[k - d:x - d])
        if len(ne):
            return k + int(ne[-1]) + 1
        x = k
    return x


def _run_fwd(a: np.ndarray, x: int, d: int) -> int:
    """The largest e >= x with a[y] == a[y - d] for all y in [x, e)."""
    n = len(a)
    while x < n:
        k = min(n, x + 4096)
        ne = np.flatnonzero(a[x:k] != a[x - d:k - d])
        if len(ne):
            return x + int(ne[0])
        x = k
    return x


def long_matches(a: np.ndarray, rate: int = LDM_RATE, maxdist: int = LDM_MAXDIST):
    """The candidate matches (s, e, d) of a chunk.  Matches that come out equal (the windows of two anchors on one
    diagonal inside one equal run) are listed once: they select the same."""
    pos, fp = anchors(a, rate)
    if len(pos) < 2:
        return []
    order = np.lexsort((pos, fp))
    sp, sf = pos[order], fp[order]
    same = np.flatnonzero((sf[1:] == sf[:-1]) & (sp[1:] - sp[:-1] <= maxdist)) + 1
    A, C = sp[same], sp[same - 1]
    w = np.arange(LDM_WINDOW) - (LDM_WINDOW - 1)
    ok = (a[A[:, None] + w] == a[C[:, None] + w]).all(axis=1)
    A, D = A[ok], A[ok] - C[ok]
    out, last = [], {}
    for i in np.argsort(A, kind="stable"):
        x, d = int(A[i]), int(D[i])
        m = last.get(d)
        if m and m[0] <= x - (LDM_WINDOW - 1) and x < m[1]:
            continue
        s = _run_back(a, x - (LDM_WINDOW - 1), d, d)
        e = _run_fwd(a, x + 1, d)
        last[d] = (s, e)
        out.append((s, e, d))
    return out


def select(matches):
    """The kept [s', e, d) in position order."""
    cur, kept = 0, []
    for s, e, d in sorted(matches, key=lambda m: (m[0], -m[1], m[2])):
        s2 = max(s, cur)
        if e - s2 >= LDM_MINMATCH:
            kept.append((s2, e, d))
            cur = e
    return kept


def _constant(blk: bytes) -> bool:
    return len(blk) > 0 and blk.count(blk[:1]) == len(blk)


def block_spans(data: bytes, rate: int = LDM_RATE):
    """Per 128 KiB block of the chunk: its long spans (start in the block, length, offset)."""
    a = np.frombuffer(data, np.uint8)
    nb = max(1, (len(data) + ZFRAME_BLOCK - 1) // ZFRAME_BLOCK)
    spans = [[] for _ in range(nb)]
    const = [_constant(data[b * ZFRAME_BLOCK:(b + 1) * ZFRAME_BLOCK]) for b in range(nb)]
    for s, e, d in select(long_matches(a, rate)):
        for b in range(s // ZFRAME_BLOCK, (e - 1) // ZFRAME_BLOCK + 1):
            ps, pe = max(s, b * ZFRAME_BLOCK), min(e, (b + 1) * ZFRAME_BLOCK)
            if not const[b] and pe - ps >= LZ_MINMATCH:
                spans[b].append((ps - b * ZFRAME_BLOCK, pe - ps, d))
    return spans


def lz_parse_spans(blk: bytes, spans, hbits: int = LZ_HBITS, tile: int = LZ_TILE, minmatch: int = LZ_MINMATCH):
    """zstd_lz_ref.lz_parse with long spans (start, length, offset), in order -> (literals, sequences)."""
    blk = bytes(blk)
    a = np.frombuffer(blk, np.uint8)
    S = len(blk)
    cand = lz_candidates(a, hbits, tile)
    ok = cand >= 0
    if len(cand):
        c, i = np.maximum(cand, 0), np.arange(len(cand))
        for k in range(minmatch):
            ok &= (i + k < S) & (a[np.minimum(c + k, S - 1)] == a[np.minimum(i + k, S - 1)])
    where = np.flatnonzero(ok).tolist()
    lits, seqs = [], []
    pos = run = j = 0
    for ss, sl, sd in list(spans) + [(S, 0, 0)]:
        while True:
            while j < len(where) and where[j] < pos:
                j += 1
            if j == len(where) or where[j] >= ss:
                break
            m = where[j]
            c = int(cand[m])
            L = minmatch
            while m + L + 16 <= S and blk[c + L: c + L + 16] == blk[m + L: m + L + 16]:
                L += 16
            while m + L < S and blk[c + L] == blk[m + L]:
                L += 1
            L = min(L, ss - m)
            if L < minmatch:
                pos = m + 1
                continue
            lits.append(blk[run:m])
            seqs.append((m - run, L, m - c))
            pos = run = m + L
        if sl:
            lits.append(blk[run:ss])
            seqs.append((ss - run, sl, sd))
            pos = run = ss + sl
    lits.append(blk[run:])
    return b"".join(lits), seqs


def zstd_frame_lzl(data: bytes, rate: int = LDM_RATE) -> bytes:
    """zstd_huf_ref.zstd_frame_lzh's frame in which a block with long spans takes its span parse's content when that
    is smaller: every block is at most its _lzh block."""
    data = bytes(data)
    out = bytearray(b"\x28\xb5\x2f\xfd\xe0" + len(data).to_bytes(8, "little"))
    nb = max(1, (len(data) + ZFRAME_BLOCK - 1) // ZFRAME_BLOCK)
    spans = block_spans(data, rate)
    for b in range(nb):
        blk = data[b * ZFRAME_BLOCK:(b + 1) * ZFRAME_BLOCK]
        last = int(b + 1 == nb)
        if _constant(blk):
            out += (last | 1 << 1 | len(blk) << 3).to_bytes(3, "little") + blk[:1]
            continue
        body = block_content_lzh(*lz_parse(blk)) if blk else blk
        if spans[b]:
            alt = block_content_lzh(*lz_parse_spans(blk, spans[b]))
            if len(alt) < len(body):
                body = alt
        if len(body) < len(blk):
            out += (last | 2 << 1 | len(body) << 3).to_bytes(3, "little") + body
        else:
            out += (last | len(blk) << 3).to_bytes(3, "little") + blk
    return bytes(out)


def blob_encode_lzl(data: bytes) -> bytes:
    """blob_encode with zstd_frame_lzl as the compressed payload (kept only when smaller than the raw bytes)."""
    import zlib
    data = bytes(data)
    if data:
        fr = zstd_frame_lzl(data)
        if len(fr) < len(data):
            return BLOB_MAGIC_COMPRESSED + zlib.crc32(fr).to_bytes(4, "little") + fr
    return BLOB_MAGIC_UNCOMPRESSED + zlib.crc32(data).to_bytes(4, "little") + data


# -- test data ---------------------------------------------------------------------------------------------------------
def repeated_image(base: np.ndarray, copies: int = 4, edits: int = 2000, seed: int = 1) -> np.ndarray:
    """`copies` copies of `base` back to back with `edits` random bytes changed at random places: repeats one copy
    apart, far beyond one block."""
    rng = np.random.default_rng(seed)
    out = np.tile(np.asarray(base, np.uint8), copies)
    out[rng.integers(0, len(out), edits)] = rng.integers(0, 256, edits, dtype=np.uint8)
    return out
