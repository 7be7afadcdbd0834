"""Restatement of the raw Deflate streams (RFC 1951) pbsgpu_deflate_batch writes (K9a's Deflate parse + K15 in
csrc/deflate.cu), in pure Python.  Test infrastructure: the GPU output is compared with it byte for byte, and zlib's
and GNU gzip's inflaters check it (tests/test_deflate_cpu.py).  csrc/deflate.cuh holds the same constants.

A range is cut into SEGMENT-byte segments, each parsed and coded on its own (no match reaches an earlier segment).
Per segment the encoder costs three forms and writes the smallest, stored then fixed on ties:
  stored   ceil(S / 65535) stored blocks (BTYPE 00), the last one partial;
  fixed    one BTYPE 01 block;
  dynamic  one BTYPE 10 block with the segment's own codes.
A segment's cost counts its end: the last segment of the stream carries BFINAL and is padded to a byte; any other
segment in fixed or dynamic form is followed by an empty non-final stored block (stored forms end byte-aligned).
An empty stream is the empty fixed block 03 00; an empty piece followed by more of the stream is no bytes at all."""
from __future__ import annotations

import numpy as np

from zstd_lz_ref import LZ_HBITS, LZ_MINMATCH, LZ_TILE, lz_candidates

SEGMENT = 128 * 1024      # bytes per independently coded segment
WINDOW = 32768            # largest match distance
MAX_MATCH = 258           # longest match
STORED_MAX = 65535        # bytes per stored block
LIT_MAXBITS = 15          # longest code of the lit/len and distance codes
CL_MAXBITS = 7            # longest code of the code-length code
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]

# RFC 1951 3.2.5: length codes 257..285 and distance codes 0..29 (base, extra bits)
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_BITS = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_BITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def bound(n: int) -> int:
    """pbsgpu_deflate_bound: every stream of n bytes fits (a segment is never larger than its stored form)."""
    return n + 15 * ((n + SEGMENT - 1) // SEGMENT) + 2


def len_code(L: int) -> int:
    return 285 if L == 258 else 257 + max(c for c in range(28) if LEN_BASE[c] <= L)


def dist_code(d: int) -> int:
    return max(c for c in range(30) if DIST_BASE[c] <= d)


def deflate_parse(blk: bytes):
    """K9a's greedy parse with the Deflate limits -> tokens: ints (literal bytes) and (length, distance) pairs.  A
    candidate counts only at distance <= WINDOW; a match is cut at MAX_MATCH and the parse resumes behind it."""
    blk = bytes(blk)
    a = np.frombuffer(blk, np.uint8)
    S = len(blk)
    cand = lz_candidates(a, LZ_HBITS, LZ_TILE)
    ok = np.zeros(len(cand), bool)
    if len(cand):
        i = np.arange(len(cand))
        c = np.maximum(cand, 0)
        ok = (cand >= 0) & (i - cand <= WINDOW)
        for k in range(LZ_MINMATCH):
            ok &= (i + k < S) & (a[np.minimum(c + k, S - 1)] == a[np.minimum(i + k, S - 1)])
    where = np.flatnonzero(ok).tolist()
    toks, pos, j = [], 0, 0
    while True:
        while j < len(where) and where[j] < pos:
            j += 1
        if j == len(where):
            break
        m = where[j]
        c = int(cand[m])
        L = LZ_MINMATCH
        while L < MAX_MATCH and m + L < S and blk[c + L] == blk[m + L]:
            L += 1
        toks.extend(blk[pos:m])
        toks.append((L, m - c))
        pos = m + L
    toks.extend(blk[pos:])
    return toks


def huffman_lengths(counts, limit: int):
    """K10's construction: present symbols in (count, symbol) order; two-queue Huffman where each step joins the two
    smallest fronts, a leaf before a node of equal count; counts halved (rounding up) until the longest code fits
    `limit`.  One present symbol gets length 1."""
    cnt = list(counts)
    n = len(cnt)
    present = [s for s in range(n) if cnt[s]]
    lengths = [0] * n
    if len(present) == 1:
        lengths[present[0]] = 1
    if len(present) <= 1:
        return lengths
    while True:
        order = sorted(present, key=lambda s: (cnt[s], s))
        m = len(order)
        w = [cnt[s] for s in order] + [0] * (m - 1)
        parent = [0] * (2 * m - 1)
        i, j, nxt = 0, m, m
        for _ in range(m - 1):
            pick = []
            for _ in range(2):
                if i < m and (j >= nxt or w[i] <= w[j]):
                    pick.append(i); i += 1
                else:
                    pick.append(j); j += 1
            w[nxt] = w[pick[0]] + w[pick[1]]
            parent[pick[0]] = parent[pick[1]] = nxt
            nxt += 1
        depth = [0] * (2 * m - 1)
        for k in range(2 * m - 3, -1, -1):
            depth[k] = depth[parent[k]] + 1
        if max(depth[:m]) <= limit:
            for k, s in enumerate(order):
                lengths[s] = depth[k]
            return lengths
        cnt = [(c + 1) >> 1 for c in cnt]


def canonical(lengths):
    """RFC 1951 3.2.2 codes, bit-reversed for an LSB-first writer."""
    mx = max(lengths) if lengths else 0
    bl = [0] * (mx + 1)
    for ln in lengths:
        if ln:
            bl[ln] += 1
    nxt, code = [0] * (mx + 2), 0
    for b in range(1, mx + 1):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for ln in lengths:
        if ln:
            c = nxt[ln]
            nxt[ln] += 1
            out.append(int(format(c, f"0{ln}b")[::-1], 2))
        else:
            out.append(0)
    return out


def cl_runs(lengths):
    """Greedy run-length coding of the code lengths: (symbol, extra value, extra bits) triples."""
    out, i, n = [], 0, len(lengths)
    while i < n:
        v = lengths[i]
        r = 1
        while i + r < n and lengths[i + r] == v:
            r += 1
        if v == 0 and r >= 11:
            k = min(r, 138); out.append((18, k - 11, 7)); i += k
        elif v == 0 and r >= 3:
            out.append((17, r - 3, 3)); i += r
        else:
            out.append((v, 0, 0)); i += 1; r -= 1
            while v and r >= 3:
                k = min(r, 6); out.append((16, k - 3, 2)); i += k; r -= k
    return out


class Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def add(self, v: int, nb: int):
        self.acc |= v << self.n
        self.n += nb
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def align(self):
        if self.n:
            self.out.append(self.acc & 0xFF)
        self.acc = self.n = 0


def _symbols(toks, lit_len, lit_code, dist_len, dist_code_, bits: Bits | None):
    """Bits of the token stream and EOB under the given codes (written to `bits` when given)."""
    total = 0
    for t in toks:
        if isinstance(t, tuple):
            L, d = t
            lc, dc = len_code(L), dist_code(d)
            eb, db = LEN_BITS[lc - 257], DIST_BITS[dc]
            total += lit_len[lc] + eb + dist_len[dc] + db
            if bits:
                bits.add(lit_code[lc], lit_len[lc]); bits.add(L - LEN_BASE[lc - 257], eb)
                bits.add(dist_code_[dc], dist_len[dc]); bits.add(d - DIST_BASE[dc], db)
        else:
            total += lit_len[t]
            if bits:
                bits.add(lit_code[t], lit_len[t])
    if bits:
        bits.add(lit_code[256], lit_len[256])
    return total + lit_len[256]


def dynamic_codes(toks):
    """The dynamic block's codes and header fields, as K15's code warp builds them."""
    lit_cnt, dist_cnt = [0] * 286, [0] * 30
    for t in toks:
        if isinstance(t, tuple):
            lit_cnt[len_code(t[0])] += 1
            dist_cnt[dist_code(t[1])] += 1
        else:
            lit_cnt[t] += 1
    lit_cnt[256] += 1
    lit_len = huffman_lengths(lit_cnt, LIT_MAXBITS)
    dist_len = huffman_lengths(dist_cnt, LIT_MAXBITS)
    hlit = max(257, max(s for s in range(286) if lit_len[s]) + 1)
    if any(dist_len):
        hdist = max(s for s in range(30) if dist_len[s]) + 1
    else:
        dist_len[0] = 1
        hdist = 1
    runs = cl_runs(lit_len[:hlit] + dist_len[:hdist])
    cl_cnt = [0] * 19
    for s, _, _ in runs:
        cl_cnt[s] += 1
    cl_len = huffman_lengths(cl_cnt, CL_MAXBITS)
    hclen = 19
    while hclen > 4 and cl_len[CL_ORDER[hclen - 1]] == 0:
        hclen -= 1
    return lit_len, dist_len, hlit, hdist, runs, cl_len, hclen


def encode_segment(blk: bytes, final: bool, stats: dict | None = None) -> bytes:
    """One segment's bytes (see the module docstring)."""
    S = len(blk)
    nstored = (S + STORED_MAX - 1) // STORED_MAX
    stored_bits = 40 * nstored + 8 * S
    toks = deflate_parse(blk)
    fixed_lit_code, fixed_dist_code = canonical(FIXED_LIT), canonical(FIXED_DIST)
    fixed_bits = 3 + _symbols(toks, FIXED_LIT, fixed_lit_code, FIXED_DIST, fixed_dist_code, None)
    lit_len, dist_len, hlit, hdist, runs, cl_len, hclen = dynamic_codes(toks)
    lit_code, dcode, cl_code = canonical(lit_len), canonical(dist_len), canonical(cl_len)
    hdr_bits = 3 + 14 + 3 * hclen + sum(cl_len[s] + nb for s, _, nb in runs)
    dyn_bits = hdr_bits + _symbols(toks, lit_len, lit_code, dist_len, dcode, None)

    def total(b):   # bits of a fixed or dynamic form with its end
        return (b + 7) // 8 * 8 if final else (b + 3 + 7) // 8 * 8 + 32

    costs = [stored_bits, total(fixed_bits), total(dyn_bits)]
    form = costs.index(min(costs))
    if stats is not None:
        stats.setdefault("forms", set()).add(("stored", "fixed", "dynamic")[form])
        if form == 2:
            stats.setdefault("cl", set()).update(s for s, _, _ in runs if s >= 16)
            stats["maxbits"] = max(stats.get("maxbits", 0), max(lit_len), max(dist_len))
            stats["cl_maxbits"] = max(stats.get("cl_maxbits", 0), max(cl_len))
    w = Bits()
    if form == 0:
        for k in range(nstored):
            part = blk[k * STORED_MAX:(k + 1) * STORED_MAX]
            w.add(int(final and k + 1 == nstored), 3)
            w.align()
            w.out += len(part).to_bytes(2, "little") + (len(part) ^ 0xFFFF).to_bytes(2, "little") + part
        return bytes(w.out)
    w.add(int(final), 1)
    if form == 1:
        w.add(1, 2)
        _symbols(toks, FIXED_LIT, fixed_lit_code, FIXED_DIST, fixed_dist_code, w)
    else:
        w.add(2, 2)
        w.add(hlit - 257, 5); w.add(hdist - 1, 5); w.add(hclen - 4, 4)
        for k in range(hclen):
            w.add(cl_len[CL_ORDER[k]], 3)
        for s, v, nb in runs:
            w.add(cl_code[s], cl_len[s]); w.add(v, nb)
        _symbols(toks, lit_len, lit_code, dist_len, dcode, w)
    if not final:
        w.add(0, 3)
        w.align()
        w.out += b"\x00\x00\xff\xff"
    w.align()
    return bytes(w.out)


def deflate(data: bytes, more: bool = False, stats: dict | None = None) -> bytes:
    """The raw Deflate stream of `data`; with `more`, a piece that a later piece continues (len a multiple of
    SEGMENT): no BFINAL and a byte-aligned end, so the pieces' concatenation is the one-piece stream."""
    data = bytes(data)
    if not data:
        return b"" if more else b"\x03\x00"
    nseg = (len(data) + SEGMENT - 1) // SEGMENT
    return b"".join(encode_segment(data[k * SEGMENT:(k + 1) * SEGMENT], not more and k + 1 == nseg, stats)
                    for k in range(nseg))


def fib_weighted(n: int, seed: int = 3) -> bytes:
    """Bytes drawn with probability 2^-L per symbol, where the number of symbols with length L (15 down to 2) follows
    the Fibonacci numbers, over shuffled byte values.  The parse still finds matches, but the lit/len code lengths keep
    a Fibonacci-like histogram, so the code-length code needs more than 7 bits before its limit (seed 3 at 128 KiB:
    9 bits) and the halving loop of the 7-bit code runs."""
    fib = [1, 1]
    while len(fib) < 20:
        fib.append(fib[-1] + fib[-2])
    lens = []
    for L in range(15, 1, -1):
        lens += [L] * max(1, fib[L] // 8 if L > 8 else 1)
    lens = lens[:256]
    rng = np.random.default_rng(seed)
    p = np.zeros(256)
    p[rng.permutation(256)[:len(lens)]] = 2.0 ** -np.array(lens)
    return bytes(rng.choice(256, size=n, p=p / p.sum()).astype(np.uint8))
