"""Restatement of the raw Deflate streams pbsgpu_deflate_batch_lzc writes (K16's DEFLATE instantiation in
csrc/zchain.cu, then K15 in csrc/deflate.cu) in numpy / pure Python.  Test infrastructure: the GPU output is compared
with it byte for byte, and zlib's and GNU gzip's inflaters check it (tests/test_deflate_chain_cpu.py).

Everything but the parse is tests/deflate_ref.py's: 128 KiB segments coded independently, the same `more` pieces, the
smallest of the stored, fixed and dynamic forms (stored then fixed on ties), the same segment ends and BFINAL, and 03 00
for the empty stream.  Each segment is parsed on its own, as one chunk of one block:
  prev(i)   for i <= S - DCH_MINMATCH: the largest j < i of the same segment whose DCH_MINMATCH bytes equal i's (exact
            byte equality).
  best(i)   among the first DCH_DEPTH chain entries j = prev(i), prev(prev(i)), ... with i - j <= WINDOW (32768), the
            longest match, extended to min(MAX_MATCH, S - i); ties go to the nearer entry.  The source may overlap i.
  parse     from the segment's first position: at a match m, while best(m + 1) exists and its gain is larger than
            best(m)'s by more than DCH_MARGIN, m becomes a literal and the parse moves on (at most DCH_LAZY times);
            gain = 4 L - the extra bits of the distance's code.  Then the match is taken and the parse jumps past it.
            After LZ_MAX_SEQ matches the rest of the segment is literals (a segment of 3-byte matches could hold more
            sequences than K15's per-segment sequence scratch).
The constants define the output bytes; csrc/zchain.cuh holds the same values, DESIGN.md K16d the sweep they come from."""
from __future__ import annotations

from bisect import bisect_left
from unittest import mock

import numpy as np

import deflate_ref as dr

DCH_MINMATCH = 3   # chain key: 3 bytes, the shortest match
DCH_DEPTH = 32     # chain entries searched per position
DCH_LAZY = 2       # positions the parse may move on from a match
DCH_MARGIN = 4     # gain a later match must exceed the current one's by
LZ_MAX_SEQ = 32768   # sequences per segment (zlz.cuh)

SEGMENT, WINDOW, MAX_MATCH = dr.SEGMENT, dr.WINDOW, dr.MAX_MATCH


def dist_extra(o: int) -> int:
    """Extra bits of the distance code of offset o (RFC 1951 3.2.5)."""
    return max(0, (o - 1).bit_length() - 2) if o > 1 else 0


def gain(L: int, o: int) -> int:
    return 4 * L - dist_extra(o)


def _words(a: np.ndarray) -> np.ndarray:
    """w[p] = the 8 bytes at p as a little-endian u64 (zeros past the end), for every p < len(a)."""
    n = len(a)
    pad = np.zeros((n + 15) // 8 * 8, np.uint8)
    pad[:n] = a
    return np.lib.stride_tricks.as_strided(pad.view("<u8"), shape=(max(n, 1),), strides=(1,))


def _match_len(w: np.ndarray, i: np.ndarray, j: np.ndarray, lim: np.ndarray) -> np.ndarray:
    """min(lim, the common length of the bytes at i and at j) per element, 8 bytes per step."""
    L = np.zeros(len(i), np.int64)
    act = np.flatnonzero(lim > 0)
    while len(act):
        x = w[i[act] + L[act]] ^ w[j[act] + L[act]]
        eq = x == 0
        low = x & (~x + np.uint64(1))
        L[act] += np.where(eq, 8, np.log2(np.where(eq, 1, low).astype(np.float64)).astype(np.int64) // 8)
        act = act[eq & (L[act] < lim[act])]
    return np.minimum(L, lim)


def best_all(data, depths=(DCH_DEPTH,), minmatch: int = DCH_MINMATCH, too_far: int = 0) -> dict:
    """best(i) of every position of the stream (segments as above) for each DEPTH in `depths`:
    {depth: (length, offset)} int64 arrays, length 0 where there is no match.  too_far > 0 (the sweep's zlib-like
    rule, not part of the format): a best(i) of 3 bytes farther back than too_far counts as no match."""
    a = np.frombuffer(bytes(data), np.uint8)
    n = len(a)
    pos = np.arange(n, dtype=np.int64)
    end = np.minimum((pos // SEGMENT + 1) * SEGMENT, n)
    keyed = np.flatnonzero(pos + minmatch <= end)
    prev = np.full(n + 1, -1, np.int64)
    if len(keyed):
        key = (keyed // SEGMENT).astype(np.uint64) << np.uint64(32)
        for k in range(minmatch):
            key |= a[keyed + k].astype(np.uint64) << np.uint64(8 * k)
        order = keyed[np.argsort(key, kind="stable")]
        ks = np.sort(key, kind="stable")
        same = ks[1:] == ks[:-1]
        prev[order[1:][same]] = order[:-1][same]
    w = _words(a)
    i = keyed
    lim = np.minimum(MAX_MATCH, end[i] - i)
    bl = np.zeros(len(i), np.int64)
    bo = np.zeros(len(i), np.int64)
    j = prev[i]
    live = np.ones(len(i), bool)   # the walk goes on: chain entries left and the longest possible not yet found
    out = {}
    for k in range(max(depths)):
        live &= (j >= 0) & (i - j <= WINDOW)
        v = np.flatnonzero(live)
        if len(v):
            L = _match_len(w, i[v], j[v], lim[v])
            up = L > bl[v]
            bl[v[up]] = L[up]
            bo[v[up]] = i[v[up]] - j[v[up]]
            live[v[bl[v] == lim[v]]] = False
            j = np.where(live, prev[np.maximum(j, 0)], -1)
        if k + 1 in depths:
            Ls, Os = np.zeros(n, np.int64), np.zeros(n, np.int64)
            Ls[i], Os[i] = bl, bo
            if too_far:
                far = (Ls == 3) & (Os > too_far)
                Ls[far], Os[far] = 0, 0
            out[k + 1] = (Ls, Os)
    for d in depths:
        if d not in out:   # a stream with no chain entries
            out[d] = (np.zeros(n, np.int64), np.zeros(n, np.int64))
    return out


def parse(L: list, O: list, lo: int, hi: int, lazy: int = DCH_LAZY, margin: int = DCH_MARGIN):
    """The lazy parse of segment [lo, hi) from best() lists -> matches [(position, length, offset)]."""
    hits = (np.flatnonzero(np.asarray(L[lo:hi])) + lo).tolist()
    seqs, i = [], lo
    while len(seqs) < LZ_MAX_SEQ:
        k = bisect_left(hits, i)
        if k == len(hits):
            break
        m = hits[k]
        l, o = L[m], O[m]
        for _ in range(lazy):
            if m + 1 >= hi or not L[m + 1] or gain(L[m + 1], O[m + 1]) <= gain(l, o) + margin:
                break
            m += 1
            l, o = L[m], O[m]
        seqs.append((m, l, o))
        i = m + l
    return seqs


def tokens(d: bytes, lo: int, hi: int, seqs) -> list:
    """deflate_ref's token list (literal ints and (length, distance) pairs) of segment [lo, hi)."""
    toks, run = [], lo
    for m, l, o in seqs:
        toks.extend(d[run:m])
        toks.append((l, o))
        run = m + l
    toks.extend(d[run:hi])
    return toks


def deflate(data, more: bool = False, stats: dict | None = None, depth: int = DCH_DEPTH, lazy: int = DCH_LAZY,
            margin: int = DCH_MARGIN, minmatch: int = DCH_MINMATCH, too_far: int = 0) -> bytes:
    """deflate_ref.deflate with the chain parse: the raw Deflate stream of `data` (a piece continued by a later one
    with `more`).  `stats["lazy"]` / `stats["refused"]` count the lazy steps taken and those the margin refused."""
    d = bytes(data)
    if not d:
        return b"" if more else b"\x03\x00"
    L, O = (x.tolist() for x in best_all(d, (depth,), minmatch, too_far)[depth])
    nseg = (len(d) + SEGMENT - 1) // SEGMENT
    out = []
    for k in range(nseg):
        lo, hi = k * SEGMENT, min(len(d), (k + 1) * SEGMENT)
        seqs = parse(L, O, lo, hi, lazy, margin)
        if stats is not None:
            _count_lazy(L, O, lo, hi, seqs, lazy, margin, stats)
        toks = tokens(d, lo, hi, seqs)
        with mock.patch.object(dr, "deflate_parse", lambda blk: toks):
            out.append(dr.encode_segment(d[lo:hi], not more and k + 1 == nseg, stats))
    return b"".join(out)


def _count_lazy(L, O, lo, hi, seqs, lazy, margin, stats):
    """Lazy steps taken (a match starts one or more positions after the first hit it came from) and refused (the next
    position had a match, but not one better by more than the margin)."""
    i = lo
    for m, l, o in seqs:
        first = next(x for x in range(i, m + 1) if L[x])
        stats["lazy"] = stats.get("lazy", 0) + (m - first)
        if m - first < lazy and m + 1 < hi and L[m + 1]:
            stats["refused"] = stats.get("refused", 0) + 1
        i = m + l
