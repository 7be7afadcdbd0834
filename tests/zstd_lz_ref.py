"""Restatement of the compressed DataBlob format with a match stage (pbsgpu_blob_encode_batch_lz, K9 in csrc/zlz.cu)
in numpy / pure Python, plus a seeded text-like corpus for it.  Test infrastructure: the GPU output is compared with it
byte for byte, and libzstd's decoder checks it (tests/test_zstd_lz_cpu.py).  The RLE / raw framing and the DataBlob
layout it builds on are oracle/pyref.py's."""
from __future__ import annotations

import numpy as np

from oracle.pyref import BLOB_MAGIC_COMPRESSED, BLOB_MAGIC_UNCOMPRESSED, ZFRAME_BLOCK

# -- compressed blocks with an LZ77 match stage (K9, csrc/zlz.cu) ------------------------------------------------------
# Per 128 KiB block of a chunk (the K8 grid): a constant block is an RLE_Block; otherwise a greedy LZ77 parse inside the
# block, Raw_Literals and a sequences section in Predefined_Mode (RFC 8878 3.1.1.3), kept when it is smaller than the
# block, else a Raw_Block.  The three constants define the output bytes (DESIGN.md K9 has the table they were chosen
# from); csrc/zlz.cuh holds the same values.
LZ_HBITS = 13        # hash table of 2^13 positions
LZ_TILE = 256        # positions looked up before any of them is inserted
LZ_MINMATCH = 4      # shortest match

# predefined distributions (RFC 8878 3.1.1.3.2.2); -1 = "less than 1" (one cell at the top of the table)
LL_NORM = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_NORM = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_NORM = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
LL_LOG, ML_LOG, OF_LOG = 6, 6, 5
# Literals_Length / Match_Length codes: baseline and extra bits (RFC 8878 3.1.1.3.2.1.1)
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387,
                                 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]


def fse_table(norm, log):
    """Decoding table of a normalized distribution (RFC 8878 4.1.1): symbol, Number_of_Bits and Baseline of every state,
    plus the encoder's view of it: enc[s][x] = the state of symbol s whose range [Baseline, + 2^Number_of_Bits) holds x,
    i.e. the state to be in when the decoder must read s and then go to state x.  The ranges of one symbol's states
    partition [0, 2^log), so enc is complete."""
    size = 1 << log
    sym = [0] * size
    high = size - 1
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
    pos, step = 0, (size >> 1) + (size >> 3) + 3
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    nxt = [1 if c == -1 else c for c in norm]
    nb, base = [0] * size, [0] * size
    for u in range(size):
        x = nxt[sym[u]]
        nxt[sym[u]] += 1
        nb[u] = log - (x.bit_length() - 1)
        base[u] = (x << nb[u]) - size
    enc = [[-1] * size for _ in norm]
    for u in range(size):
        for x in range(base[u], base[u] + (1 << nb[u])):
            enc[sym[u]][x] = u
    return sym, nb, base, enc


_FSE = {}


def _tables():
    if not _FSE:
        _FSE["ll"] = fse_table(LL_NORM, LL_LOG)
        _FSE["ml"] = fse_table(ML_NORM, ML_LOG)
        _FSE["of"] = fse_table(OF_NORM, OF_LOG)
    return _FSE["ll"], _FSE["ml"], _FSE["of"]


def _code(bases, v):
    c = 0
    while c + 1 < len(bases) and bases[c + 1] <= v:
        c += 1
    return c


def seq_codes(ll: int, ml: int, off: int):
    """(code, extra value, extra bits) for Literals_Length, Match_Length and Offset; Offset_Value = off + 3."""
    lc, mc = _code(LL_BASE, ll), _code(ML_BASE, ml)
    ov = off + 3
    oc = ov.bit_length() - 1
    return (lc, ll - LL_BASE[lc], LL_BITS[lc]), (mc, ml - ML_BASE[mc], ML_BITS[mc]), (oc, ov - (1 << oc), oc)


def seq_bitstream(seqs) -> bytes:
    """The sequences bitstream (RFC 8878 3.1.1.3.2.2) of a non-empty list of (literal length, match length, offset), all
    three tables predefined.  Written forward, read backward: the last sequence's extra bits (LL, ML, OF) come first,
    then per earlier sequence the state bits (OF, ML, LL) that lead to its successor's states and its extra bits, then
    the first sequence's states (ML, OF, LL) and the end mark.  The last sequence's states are enc[code][0]."""
    tl, tm, to = _tables()
    codes = [seq_codes(*s) for s in seqs]
    out = bytearray()
    acc = nacc = 0

    def add(v, n):
        nonlocal acc, nacc
        acc |= v << nacc
        nacc += n
        while nacc >= 8:
            out.append(acc & 0xFF)
            acc >>= 8
            nacc -= 8

    (lc, lv, lb), (mc, mv, mb), (oc, ov, ob) = codes[-1]
    st = [tl[3][lc][0], tm[3][mc][0], to[3][oc][0]]
    add(lv, lb); add(mv, mb); add(ov, ob)
    for k in range(len(codes) - 2, -1, -1):
        (lc, lv, lb), (mc, mv, mb), (oc, ov, ob) = codes[k]
        for t, tab, c in ((2, to, oc), (1, tm, mc), (0, tl, lc)):
            u = tab[3][c][st[t]]
            add(st[t] - tab[2][u], tab[1][u])
            st[t] = u
        add(lv, lb); add(mv, mb); add(ov, ob)
    add(st[1], ML_LOG); add(st[2], OF_LOG); add(st[0], LL_LOG); add(1, 1)
    if nacc:
        out.append(acc & 0xFF)
    return bytes(out)


def compressed_block(literals: bytes, seqs) -> bytes:
    """Block_Content of a Compressed_Block: Raw_Literals_Block (1-, 2- or 3-byte header for sizes <= 31, <= 4095,
    larger) + Sequences_Section (count in 1, 2 or 3 bytes, Symbol_Compression_Modes 0 = all predefined; a block without
    sequences is the single 0 byte)."""
    n_lit, n = len(literals), len(seqs)
    if n_lit <= 31:
        hdr = bytes([n_lit << 3])
    elif n_lit <= 4095:
        hdr = ((n_lit << 4) | 0b0100).to_bytes(2, "little")
    else:
        hdr = ((n_lit << 4) | 0b1100).to_bytes(3, "little")
    if n == 0:
        return hdr + bytes(literals) + b"\0"
    if n < 128:
        cnt = bytes([n])
    elif n < 0x7F00:
        cnt = bytes([(n >> 8) + 0x80, n & 0xFF])
    else:
        cnt = b"\xff" + (n - 0x7F00).to_bytes(2, "little")
    return hdr + bytes(literals) + cnt + b"\0" + seq_bitstream(seqs)


def lz_candidates(blk: np.ndarray, hbits: int = LZ_HBITS, tile: int = LZ_TILE) -> np.ndarray:
    """cand(i) for i <= S-4: the largest j in an earlier tile of the block with h(j) == h(i), else -1.
    key(i) = u32 LE at i, h(i) = (key(i) * 0x9E3779B1 mod 2^32) >> (32 - hbits)."""
    nk = len(blk) - 3
    if nk <= 0:
        return np.zeros(0, np.int64)
    b = blk.astype(np.uint32)
    key = b[:nk] | b[1:nk + 1] << 8 | b[2:nk + 2] << 16 | b[3:nk + 3] << 24
    h = ((key.astype(np.uint64) * 0x9E3779B1) & 0xFFFFFFFF) >> (32 - hbits)
    pos = np.arange(nk, dtype=np.int64)
    sk = h.astype(np.int64) * nk + pos                     # (hash, position), sorted
    order = np.argsort(sk, kind="stable")
    sk = sk[order]
    q = np.searchsorted(sk, h.astype(np.int64) * nk + pos // tile * tile, side="left") - 1
    qc = np.maximum(q, 0)
    ok = (q >= 0) & (sk[qc] // nk == h.astype(np.int64))
    return np.where(ok, order[qc], -1)


def lz_parse(blk: bytes, hbits: int = LZ_HBITS, tile: int = LZ_TILE, minmatch: int = LZ_MINMATCH):
    """Greedy parse of one block -> (literals, [(literal length, match length, offset)]).  A match at i: cand(i) exists
    and the longest common extension of cand(i) and i inside the block is >= minmatch (it may overlap i)."""
    blk = bytes(blk)
    a = np.frombuffer(blk, np.uint8)
    S = len(blk)
    cand = lz_candidates(a, hbits, tile)
    match_at = np.zeros(len(cand), bool)
    if len(cand):
        c = np.maximum(cand, 0)
        i = np.arange(len(cand))
        ok = cand >= 0
        for k in range(minmatch):              # the first minmatch bytes, inside the block
            inside = i + k < S
            ok &= inside & (a[np.minimum(c + k, S - 1)] == a[np.minimum(i + k, S - 1)])
        match_at = ok
    where = np.flatnonzero(match_at).tolist()
    lits, seqs = [], []
    pos, j = 0, 0
    while True:
        while j < len(where) and where[j] < pos:
            j += 1
        if j == len(where):
            break
        m = where[j]
        c = int(cand[m])
        L = minmatch
        while m + L + 16 <= S and blk[c + L: c + L + 16] == blk[m + L: m + L + 16]:
            L += 16
        while m + L < S and blk[c + L] == blk[m + L]:
            L += 1
        lits.append(blk[pos:m])
        seqs.append((m - pos, L, m - c))
        pos = m + L
    lits.append(blk[pos:])
    return b"".join(lits), seqs


def zstd_frame_lz(data: bytes, hbits: int = LZ_HBITS, tile: int = LZ_TILE, minmatch: int = LZ_MINMATCH) -> bytes:
    """zstd_frame_rle_raw's frame in which a block that is not constant is a Compressed_Block (Block_Type 2) of its
    greedy LZ77 parse when that is strictly smaller than the block, else a Raw_Block.  Every block is therefore at most
    as large as in zstd_frame_rle_raw."""
    data = bytes(data)
    out = bytearray(b"\x28\xb5\x2f\xfd\xe0" + len(data).to_bytes(8, "little"))
    nb = max(1, (len(data) + ZFRAME_BLOCK - 1) // ZFRAME_BLOCK)
    for b in range(nb):
        blk = data[b * ZFRAME_BLOCK:(b + 1) * ZFRAME_BLOCK]
        last = int(b + 1 == nb)
        if len(blk) > 0 and blk.count(blk[:1]) == len(blk):
            out += (last | 1 << 1 | len(blk) << 3).to_bytes(3, "little") + blk[:1]
            continue
        body = compressed_block(*lz_parse(blk, hbits, tile, minmatch)) if blk else blk
        if len(body) < len(blk):
            out += (last | 2 << 1 | len(body) << 3).to_bytes(3, "little") + body
        else:
            out += (last | len(blk) << 3).to_bytes(3, "little") + blk
    return bytes(out)


def blob_encode_lz(data: bytes) -> bytes:
    """blob_encode with zstd_frame_lz as the compressed payload (kept only when smaller than the raw bytes)."""
    import zlib
    data = bytes(data)
    if data:
        fr = zstd_frame_lz(data)
        if len(fr) < len(data):
            return BLOB_MAGIC_COMPRESSED + zlib.crc32(fr).to_bytes(4, "little") + fr
    return BLOB_MAGIC_UNCOMPRESSED + zlib.crc32(data).to_bytes(4, "little") + data


def text_corpus(nbytes: int, seed: int = 0) -> np.ndarray:
    """Deterministic compressible test data: 96 KiB stretches of a Zipf-distributed word stream (a 4096-word vocabulary
    built from syllables, with sentence ends and line breaks) alternating with 32 KiB stretches of structured records
    (log lines with a timestamp, host, service, hex id and counters)."""
    rng = np.random.default_rng(seed)
    syl = ["ka", "lo", "mi", "ne", "ru", "ta", "shi", "po", "en", "dar", "vel", "qu", "ix", "or", "am", "bel"]
    words = ["".join(rng.choice(syl, rng.integers(1, 5))) for _ in range(4096)]
    toks = [w + s for w in words for s in (" ", ". ", "\n")]               # token = word + separator
    tflat = np.frombuffer("".join(toks).encode(), np.uint8)
    tlen = np.array([len(t) for t in toks], np.int64)
    tstart = np.concatenate([[0], np.cumsum(tlen)[:-1]])
    p = 1.0 / np.arange(1, len(words) + 1)
    p /= p.sum()
    svc = ["auth", "disk", "net", "sched", "backup", "gc", "api", "cron"]
    out = np.empty(nbytes, np.uint8)
    pos, t = 0, 0
    while pos < nbytes:
        want = min(96 << 10 if t % 2 == 0 else 32 << 10, nbytes - pos)
        if t % 2 == 0:
            m = want // 5 + 16
            ids = rng.choice(len(words), m, p=p) * 3 + rng.choice(3, m, p=[0.88, 0.08, 0.04])
            L = tlen[ids]
            ends = np.cumsum(L)
            idx = np.repeat(tstart[ids] - (ends - L), L) + np.arange(int(ends[-1]))
            seg = tflat[idx][:want]
        else:
            lines = []
            size = 0
            while size < want:
                s = (f"2026-10-{rng.integers(1, 29):02d}T{rng.integers(0, 24):02d}:{rng.integers(0, 60):02d}:"
                     f"{rng.integers(0, 60):02d}.{rng.integers(0, 1000):03d}Z host-{rng.integers(0, 64):03d} "
                     f"svc={svc[rng.integers(0, 8)]} id={rng.integers(0, 1 << 32):08x} bytes={rng.integers(0, 1 << 20)} "
                     f"status={(200, 200, 200, 204, 404, 500)[rng.integers(0, 6)]}\n")
                lines.append(s)
                size += len(s)
            seg = np.frombuffer("".join(lines).encode()[:want], np.uint8)
        out[pos:pos + len(seg)] = seg
        pos += len(seg)
        t += 1
    return out
