"""Restatement of the compressed DataBlob format with zstd's entropy stage (pbsgpu_blob_encode_batch_lze, K10 in
csrc/zent.cu) in numpy / pure Python.  Test infrastructure: the GPU output is compared with it byte for byte, and
libzstd's decoder checks it (tests/test_zstd_ent_cpu.py).  The parse, the predefined-table block writer and the FSE table
construction are tests/zstd_lz_ref.py's, unchanged.

Per block that is not constant, the Block_Content is the smaller of compressed_block (the _lz content, which wins ties)
and entropy_block below; the block stays raw when neither is smaller than the block."""
from __future__ import annotations

import numpy as np

from oracle.pyref import BLOB_MAGIC_COMPRESSED, BLOB_MAGIC_UNCOMPRESSED, ZFRAME_BLOCK
from zstd_lz_ref import LZ_HBITS, LZ_MINMATCH, LZ_TILE, compressed_block, fse_table, lz_parse, seq_codes

# Largest accuracy logs the format allows for FSE_Compressed_Mode tables (RFC 8878 3.1.1.3.2.1.2) and the smallest
# one the table description can state; the longest Huffman code the literals may use (RFC 8878 4.2.1).
LL_MAXLOG, OF_MAXLOG, ML_MAXLOG = 9, 8, 9
MIN_LOG = 5
HUF_MAXBITS = 11
HUF_MAXSYMBOL = 128     # the direct 4-bit weight form lists at most 128 weights; the last symbol's weight is implied


class _Bits:
    """Bits appended LSB first (the order of every zstd bitstream, which is read from its end)."""

    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def add(self, v, n):
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def flush(self) -> bytes:
        if self.n:
            self.out.append(self.acc & 0xFF)
        return bytes(self.out)


# -- FSE_Compressed_Mode tables ----------------------------------------------------------------------------------------
def accuracy_log(n: int, distinct: int, cap: int) -> int:
    """Accuracy log of a table over n sequences with `distinct` codes present: bit_length(n) - 2 (about 4 sequences per
    state), clamped to [MIN_LOG, cap], and raised to ceil(log2(distinct)) so every present code gets a state.  DESIGN.md
    K10 has the table this rule was chosen from."""
    log = min(cap, max(MIN_LOG, n.bit_length() - 2))
    while (1 << log) < distinct:
        log += 1
    return log


def normalize(counts, log):
    """Distribution summing to 2^log with every present code >= 1 (no "less than 1" cells): start from
    max(1, floor(count * 2^log / n)); while the sum is too large, decrement the largest entry (the lowest code on
    ties); if it is too small, add the difference to the entry with the largest count (the lowest code on ties)."""
    n, size = sum(counts), 1 << log
    norm = [max(1, c * size // n) if c else 0 for c in counts]
    s = sum(norm)
    while s > size:
        k = max(range(len(norm)), key=lambda i: (norm[i], -i))
        norm[k] -= 1
        s -= 1
    if s < size:
        k = max(range(len(counts)), key=lambda i: (counts[i], -i))
        norm[k] += size - s
    return norm


def fse_description(norm, log) -> bytes:
    """FSE table description (RFC 8878 4.1.1): Accuracy_Log - 5 in 4 bits, then each code's count + 1 in a variable
    number of bits (the low values one bit shorter), a zero count followed by 2-bit repeat flags for the zero counts
    after it; it stops when the counts reach 2^log.  A count of -1 ("less than 1") takes one cell."""
    w = _Bits()
    w.add(log - MIN_LOG, 4)
    remaining, threshold, nbits = (1 << log) + 1, 1 << log, log + 1
    s, prev0 = 0, False
    while s < len(norm) and remaining > 1:
        if prev0:
            start = s
            while norm[s] == 0:
                s += 1
            while s >= start + 3:
                start += 3
                w.add(3, 2)
            w.add(s - start, 2)
        c = norm[s]
        s += 1
        mx = 2 * threshold - 1 - remaining
        remaining -= abs(c)
        c += 1
        if c >= threshold:
            c += mx
        w.add(c, nbits - (c < mx))
        prev0 = c == 1
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    return w.flush()


def table_for(codes, nsym, cap):
    """(mode, description, fse_table, log) of one of the LL / OF / ML columns: RLE_Mode when every sequence has the same
    code, else FSE_Compressed_Mode with the block's own distribution."""
    counts = np.bincount(np.asarray(codes), minlength=nsym).tolist()
    present = [c for c in range(nsym) if counts[c]]
    if len(present) == 1:
        norm = [0] * nsym
        norm[present[0]] = 1
        return 1, bytes(present), fse_table(norm, 0), 0
    log = accuracy_log(len(codes), len(present), cap)
    norm = normalize(counts, log)
    return 2, fse_description(norm, log), fse_table(norm, log), log


def seq_bitstream_tables(codes, tl, tm, to, logs) -> bytes:
    """zstd_lz_ref.seq_bitstream with the block's tables (ll, ml, of) of accuracy logs `logs` in place of the predefined
    ones; the same order of fields and the same start states for the last sequence (enc[code][0])."""
    w = _Bits()
    (lc, lv, lb), (mc, mv, mb), (oc, ov, ob) = codes[-1]
    st = [tl[3][lc][0], tm[3][mc][0], to[3][oc][0]]
    w.add(lv, lb); w.add(mv, mb); w.add(ov, ob)
    for k in range(len(codes) - 2, -1, -1):
        (lc, lv, lb), (mc, mv, mb), (oc, ov, ob) = codes[k]
        for t, tab, c in ((2, to, oc), (1, tm, mc), (0, tl, lc)):
            u = tab[3][c][st[t]]
            w.add(st[t] - tab[2][u], tab[1][u])
            st[t] = u
        w.add(lv, lb); w.add(mv, mb); w.add(ov, ob)
    w.add(st[1], logs[1]); w.add(st[2], logs[2]); w.add(st[0], logs[0]); w.add(1, 1)
    return w.flush()


def sequences_section(seqs) -> bytes:
    """Sequences_Section: the count as in compressed_block, the modes byte (LL << 6 | OF << 4 | ML << 2), the LL, OF
    and ML table descriptions in that order, and the bitstream."""
    n = len(seqs)
    if n == 0:
        return b"\0"
    if n < 128:
        cnt = bytes([n])
    elif n < 0x7F00:
        cnt = bytes([(n >> 8) + 0x80, n & 0xFF])
    else:
        cnt = b"\xff" + (n - 0x7F00).to_bytes(2, "little")
    codes = [seq_codes(*s) for s in seqs]
    ml_, dl, tl, gl = table_for([c[0][0] for c in codes], 36, LL_MAXLOG)
    mo, do, to, go = table_for([c[2][0] for c in codes], 32, OF_MAXLOG)
    mm, dm, tm, gm = table_for([c[1][0] for c in codes], 53, ML_MAXLOG)
    return cnt + bytes([ml_ << 6 | mo << 4 | mm << 2]) + dl + do + dm + seq_bitstream_tables(codes, tl, tm, to, (gl, gm, go))


# -- Huffman-coded literals --------------------------------------------------------------------------------------------
def _huffman(counts):
    """Code lengths of a two-queue Huffman build: leaves in (count, symbol) order, internal nodes in the order they are
    made, each step joins the two smallest fronts (a leaf before a node of equal count)."""
    sym = sorted((c, s) for s, c in enumerate(counts) if c)
    m = len(sym)
    w = [c for c, _ in sym] + [0] * (m - 1)
    parent = [0] * (2 * m - 1)
    i, j, nxt = 0, m, m
    for _ in range(m - 1):
        pick = []
        for _ in range(2):
            if i < m and (j >= nxt or w[i] <= w[j]):
                pick.append(i)
                i += 1
            else:
                pick.append(j)
                j += 1
        w[nxt] = w[pick[0]] + w[pick[1]]
        parent[pick[0]] = parent[pick[1]] = nxt
        nxt += 1
    depth = [0] * (2 * m - 1)
    for k in range(2 * m - 3, -1, -1):                      # a parent is made after its children
        depth[k] = depth[parent[k]] + 1
    lengths = [0] * len(counts)
    for k, (_, s) in enumerate(sym):
        lengths[s] = depth[k]
    return lengths


def huf_lengths(counts):
    """Huffman code lengths <= HUF_MAXBITS for >= 2 present symbols: while the longest code is too long, halve every
    count (rounding up, so a present symbol stays present) and build again.  The code is complete."""
    cnt = list(counts)
    while True:
        lengths = _huffman(cnt)
        if max(lengths) <= HUF_MAXBITS:
            return lengths
        cnt = [(c + 1) >> 1 for c in cnt]


def huf_codes(lengths):
    """Canonical codes the decoder derives from the weights (RFC 8878 4.2.1.3): symbols in (length descending, symbol
    ascending) order take consecutive prefixes, in units of 2^(maxbits - length)."""
    mx = max(lengths)
    codes, nxt = [0] * len(lengths), 0
    for neg, s in sorted((-ln, s) for s, ln in enumerate(lengths) if ln):
        codes[s] = nxt >> (mx + neg)
        nxt += 1 << (mx + neg)
    return codes


def huf_stream(lits: np.ndarray, codes: np.ndarray, lengths: np.ndarray) -> bytes:
    """One Huffman stream: the literals' codes from the LAST literal to the first, LSB first, then the end mark, so the
    decoder, reading from the end, meets the first literal's code first."""
    r = lits[::-1]
    ln = lengths[r].astype(np.int64)
    cd = codes[r].astype(np.int64)
    total = int(ln.sum())
    start = np.repeat(np.cumsum(ln) - ln, ln)
    j = np.arange(total) - start
    bits = np.zeros(total + 1, np.uint8)
    bits[:total] = (np.repeat(cd, ln) >> j) & 1
    bits[total] = 1
    return np.packbits(bits, bitorder="little").tobytes()


def _lit_header(kind: int, n: int) -> bytes:
    """Raw_ (kind 0) or RLE_Literals_Block (kind 1) header, Size_Format 00 / 01 / 11 for n <= 31, <= 4095, larger."""
    if n <= 31:
        return bytes([kind | n << 3])
    if n <= 4095:
        return (kind | 0b0100 | n << 4).to_bytes(2, "little")
    return (kind | 0b1100 | n << 4).to_bytes(3, "little")


def huffman_literals(lits: np.ndarray, hist) -> bytes:
    """Compressed_Literals_Block: the tree description in the direct form (header byte 127 + largest symbol, then a
    4-bit weight per symbol below it, weight = maxbits + 1 - length or 0), then one stream when the regenerated and
    compressed sizes both fit 10 bits (Size_Format 00), else four streams behind the 6-byte jump table, the first three
    holding (size + 3) / 4 literals each, with the smallest Size_Format of 01 / 10 / 11 (10 / 14 / 18 bits) that fits."""
    lengths = huf_lengths(hist)
    codes = np.array(huf_codes(lengths), np.int64)
    ln_arr = np.array(lengths, np.int64)
    mx, top = max(lengths), max(s for s in range(256) if lengths[s])
    wts = [mx + 1 - lengths[s] if lengths[s] else 0 for s in range(top)] + [0]
    tree = bytes([127 + top]) + bytes(wts[k] << 4 | wts[k + 1] for k in range(0, top, 2))
    n = len(lits)
    one = tree + huf_stream(lits, codes, ln_arr)
    if n <= 1023 and len(one) <= 1023:
        return (2 | n << 4 | len(one) << 14).to_bytes(3, "little") + one
    seg = (n + 3) // 4
    st = [huf_stream(lits[k * seg:min(n, (k + 1) * seg)], codes, ln_arr) for k in range(4)]
    body = tree + b"".join(len(s).to_bytes(2, "little") for s in st[:3]) + b"".join(st)
    c = len(body)
    if max(n, c) <= 1023:
        return (2 | 1 << 2 | n << 4 | c << 14).to_bytes(3, "little") + body
    if max(n, c) <= 16383:
        return (2 | 2 << 2 | n << 4 | c << 18).to_bytes(4, "little") + body
    return (2 | 3 << 2 | n << 4 | c << 22).to_bytes(5, "little") + body


def literals_section(lits: bytes) -> bytes:
    """RLE_Literals_Block when all literals have one value; Huffman-coded when there are >= 2 values, none above
    HUF_MAXSYMBOL, and that section is smaller than the raw one; else Raw_Literals_Block (as in compressed_block)."""
    raw = _lit_header(0, len(lits)) + lits
    if not lits:
        return raw
    a = np.frombuffer(lits, np.uint8)
    hist = np.bincount(a, minlength=256).tolist()
    if np.count_nonzero(hist) == 1:
        return _lit_header(1, len(lits)) + lits[:1]
    if int(a.max()) > HUF_MAXSYMBOL:
        return raw
    huf = huffman_literals(a, hist)
    return huf if len(huf) < len(raw) else raw


def entropy_block(lits: bytes, seqs) -> bytes:
    """Block_Content with the entropy stage: literals_section + sequences_section."""
    return literals_section(bytes(lits)) + sequences_section(seqs)


def block_content(lits: bytes, seqs) -> bytes:
    """The smaller of the _lz content (compressed_block, which wins ties) and entropy_block."""
    lz, ent = compressed_block(lits, seqs), entropy_block(lits, seqs)
    return ent if len(ent) < len(lz) else lz


def zstd_frame_lze(data: bytes, hbits: int = LZ_HBITS, tile: int = LZ_TILE, minmatch: int = LZ_MINMATCH) -> bytes:
    """zstd_lz_ref.zstd_frame_lz's frame with block_content in place of compressed_block: every block is at most its
    _lz block."""
    data = bytes(data)
    out = bytearray(b"\x28\xb5\x2f\xfd\xe0" + len(data).to_bytes(8, "little"))
    nb = max(1, (len(data) + ZFRAME_BLOCK - 1) // ZFRAME_BLOCK)
    for b in range(nb):
        blk = data[b * ZFRAME_BLOCK:(b + 1) * ZFRAME_BLOCK]
        last = int(b + 1 == nb)
        if len(blk) > 0 and blk.count(blk[:1]) == len(blk):
            out += (last | 1 << 1 | len(blk) << 3).to_bytes(3, "little") + blk[:1]
            continue
        body = block_content(*lz_parse(blk, hbits, tile, minmatch)) if blk else blk
        if len(body) < len(blk):
            out += (last | 2 << 1 | len(body) << 3).to_bytes(3, "little") + body
        else:
            out += (last | len(blk) << 3).to_bytes(3, "little") + blk
    return bytes(out)


def blob_encode_lze(data: bytes) -> bytes:
    """blob_encode with zstd_frame_lze as the compressed payload (kept only when smaller than the raw bytes)."""
    import zlib
    data = bytes(data)
    if data:
        fr = zstd_frame_lze(data)
        if len(fr) < len(data):
            return BLOB_MAGIC_COMPRESSED + zlib.crc32(fr).to_bytes(4, "little") + fr
    return BLOB_MAGIC_UNCOMPRESSED + zlib.crc32(data).to_bytes(4, "little") + data
