"""Which zstd block forms a set of frames reaches: a frame walker written from RFC 8878 alone (it shares no code with the
restatements' writers), a census of named forms over frames, the forms each blob mode must show, and seeded inputs built
to reach the rare ones.  Test infrastructure for tests/test_zstd_forms_cpu.py and tests/test_gpu_zstd_forms.py: the GPU
frames equal the restatements' byte for byte, so a census of either says which branches of K9 / K10 an input set runs.

Form names (census):
  block:raw | block:rle | block:compressed
  lit:raw/1B..3B | lit:rle/1B..3B   Raw_ / RLE_Literals_Block and its header size
  lit:huf/sf0..3                    Compressed_Literals_Block and its Size_Format (sf0: one stream)
  tree:direct | tree:fse/log5/odd   Huffman tree description form; the FSE form's accuracy log and weight-count parity
  huf:maxlen11                      the longest Huffman code is HUF_MAXBITS long
  nseq:0 | nseq:1B..3B              Number_of_Sequences and its byte form; nseq:127 / 128 / 0x7EFF / 0x7F00 at the edges
  modes:FFR                         Literals_Lengths, Offsets, Match_Lengths modes: Predefined, RLE, FSE_Compressed, Repeat
  LL:log5 | OF:log8 | ...           accuracy log of an FSE_Compressed table
"""
from __future__ import annotations

from collections import Counter
from dataclasses import dataclass
from functools import lru_cache

import numpy as np

from zstd_lz_ref import text_corpus

ZSTD_MAGIC = 0xFD2FB528
MODE_LETTER = "PRFX"                                  # Predefined, RLE, FSE_Compressed, Repeat
COLUMNS = (("LL", 35), ("OF", 31), ("ML", 52))        # column and its largest code (RFC 8878 3.1.1.3.2.1)
HUF_MAXBITS = 11                                      # the encoders' Huffman length limit (zstd_ent_ref.HUF_MAXBITS)
EDGE_COUNTS = {127: "nseq:127", 128: "nseq:128", 0x7EFF: "nseq:0x7EFF", 0x7F00: "nseq:0x7F00"}


@dataclass
class BlockInfo:
    type: int                                   # 0 raw, 1 RLE, 2 compressed
    size: int                                   # Block_Size field
    last: bool
    lit_type: int | None = None                 # 0 raw, 1 RLE, 2 compressed, 3 treeless
    lit_sf: int | None = None                   # Size_Format
    lit_hdr: int | None = None                  # literals section header bytes
    lit_regen: int | None = None
    lit_comp: int | None = None                 # compressed size (Huffman literals: tree + jump table + streams)
    lit_streams: int | None = None
    tree: str | None = None                     # "direct" or "fse"
    tree_log: int | None = None                 # accuracy log of the FSE weight table
    tree_weights: int | None = None             # number of listed weights (the last symbol's is implied)
    huf_maxlen: int | None = None               # longest Huffman code, from the weights
    nseq: int | None = None
    nseq_bytes: int | None = None               # 1, 2 or 3; 0 when nseq == 0 (a single zero byte, no modes byte)
    modes: tuple | None = None                  # (LL, OF, ML) Symbol_Compression_Modes
    logs: tuple | None = None                   # accuracy log of each column's FSE_Compressed table, else None


# -- bit readers ---------------------------------------------------------------------------------------------------------
class _Forward:
    """Bits LSB first from `pos` on (FSE table descriptions, RFC 8878 4.1.1)."""

    def __init__(self, data: bytes, pos: int):
        self.data, self.bit = data, pos * 8

    def peek(self, n: int) -> int:
        v = 0
        for k in range(n):
            b = self.bit + k
            v |= ((self.data[b >> 3] >> (b & 7)) & 1) << k
        return v

    def read(self, n: int) -> int:
        v = self.peek(n)
        self.bit += n
        return v

    def end(self) -> int:
        """The first byte after the bits read."""
        return (self.bit + 7) >> 3


def read_fse_description(data: bytes, pos: int, max_symbol: int):
    """An FSE table description at data[pos:] (RFC 8878 4.1.1) -> (accuracy log, counts, the position after it).
    Counts are normalised (-1 = "less than 1"); a zero count is followed by 2-bit repeat flags (3 = three more zeros and
    another flag)."""
    r = _Forward(data, pos)
    log = r.read(4) + 5
    remaining, threshold, nbits = (1 << log) + 1, 1 << log, log + 1
    counts, prev0 = [], False
    while remaining > 1 and len(counts) <= max_symbol:
        if prev0:
            while True:
                rep = r.read(2)
                counts += [0] * rep
                if rep != 3:
                    break
        mx = 2 * threshold - 1 - remaining
        low = r.peek(nbits - 1)
        if low < mx:
            v = low
            r.bit += nbits - 1
        else:
            v = r.read(nbits)
            if v >= threshold:
                v -= mx
        c = v - 1
        remaining -= abs(c)
        counts.append(c)
        prev0 = c == 0
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    if remaining != 1 or len(counts) > max_symbol + 1:
        raise ValueError(f"bad FSE table description at {pos}")
    return log, counts, r.end()


def fse_decoding_table(counts, log):
    """(symbol, Number_of_Bits, Baseline) of every state (RFC 8878 4.1.1)."""
    size = 1 << log
    sym = [0] * size
    high = size - 1
    for s, c in enumerate(counts):
        if c == -1:
            sym[high] = s
            high -= 1
    pos, step = 0, (size >> 1) + (size >> 3) + 3
    for s, c in enumerate(counts):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    nxt = [1 if c == -1 else c for c in counts]
    table = []
    for u in range(size):
        x = nxt[sym[u]]
        nxt[sym[u]] += 1
        nb = log - (x.bit_length() - 1)
        table.append((sym[u], nb, (x << nb) - size))
    return table


def fse_weights_decode(data: bytes) -> tuple[int, list[int]]:
    """The FSE-compressed Huffman weights (RFC 8878 4.2.1.2) of `data` (the header byte's span) -> (accuracy log,
    weights).  Two interleaved states over one backward bitstream; decoding stops when a state update reads past the
    stream's start, and the other state then gives one last weight."""
    log, counts, p = read_fse_description(data, 0, 255)
    table = fse_decoding_table(counts, log)
    stream = data[p:]
    if not stream or stream[-1] == 0:
        raise ValueError("Huffman weight stream without its end mark")
    avail = 8 * len(stream) - (8 - stream[-1].bit_length()) - 1
    used = 0

    def read(n):
        nonlocal used
        used += n
        v = 0
        for k in range(n):                                   # bit avail - used + k, zero before the stream's start
            b = avail - used + k
            if b >= 0:
                v |= ((stream[b >> 3] >> (b & 7)) & 1) << k
        return v

    st = [read(log), read(log)]
    out, t = [], 0
    while True:
        s, nb, base = table[st[t]]
        out.append(s)
        st[t] = base + read(nb)
        if used > avail:
            out.append(table[st[1 - t]][0])
            return log, out
        if len(out) > 255:
            raise ValueError("Huffman weight stream does not end")
        t = 1 - t


def _huf_maxlen(weights: list[int]) -> int:
    """Longest code of the Huffman code the decoder derives from the listed weights and the implied last one."""
    total = sum(1 << (w - 1) for w in weights if w)
    maxbits = total.bit_length()
    rest = (1 << maxbits) - total
    if total == 0 or rest & (rest - 1):
        raise ValueError("Huffman weights do not complete a code")
    last = rest.bit_length()                                  # weight of the implied symbol: log2(rest) + 1
    return maxbits + 1 - min([w for w in weights if w] + [last])


# -- sections -------------------------------------------------------------------------------------------------------
def _literals(body: bytes, info: BlockInfo) -> int:
    """Reads the Literals_Section header and tree description into info; returns the section's size."""
    b0 = body[0]
    t, sf = b0 & 3, (b0 >> 2) & 3
    info.lit_type, info.lit_sf = t, sf
    if t in (0, 1):
        if sf in (0, 2):
            h, n = 1, b0 >> 3
        elif sf == 1:
            h, n = 2, (b0 >> 4) | body[1] << 4
        else:
            h, n = 3, (b0 >> 4) | body[1] << 4 | body[2] << 12
        info.lit_hdr, info.lit_regen = h, n
        return h + (n if t == 0 else 1)
    h, w = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
    v = int.from_bytes(body[:h], "little")
    info.lit_hdr, info.lit_streams = h, 1 if sf == 0 else 4
    info.lit_regen, info.lit_comp = (v >> 4) & ((1 << w) - 1), (v >> (4 + w)) & ((1 << w) - 1)
    if t == 2:
        th = body[h]
        if th >= 128:
            nw = th - 127
            raw = body[h + 1:h + 1 + (nw + 1) // 2]
            weights = [(raw[k // 2] >> (4 if k % 2 == 0 else 0)) & 15 for k in range(nw)]
            info.tree = "direct"
        else:
            info.tree_log, weights = fse_weights_decode(body[h + 1:h + 1 + th])
            info.tree = "fse"
        info.tree_weights = len(weights)
        info.huf_maxlen = _huf_maxlen(weights)
    return h + info.lit_comp


def _sequences(sec: bytes, info: BlockInfo):
    b0 = sec[0]
    if b0 == 0:
        info.nseq, info.nseq_bytes = 0, 0
        return
    if b0 < 128:
        n, k = b0, 1
    elif b0 < 255:
        n, k = ((b0 - 128) << 8) + sec[1], 2
    else:
        n, k = sec[1] + (sec[2] << 8) + 0x7F00, 3
    info.nseq, info.nseq_bytes = n, k
    m = sec[k]
    if m & 3:
        raise ValueError("reserved bits of Symbol_Compression_Modes set")
    info.modes = (m >> 6, (m >> 4) & 3, (m >> 2) & 3)
    pos, logs = k + 1, []
    for (name, max_sym), mode in zip(COLUMNS, info.modes):
        log = None
        if mode == 1:
            pos += 1
        elif mode == 2:
            log, _, pos = read_fse_description(sec, pos, max_sym)
        logs.append(log)
    info.logs = tuple(logs)
    if pos >= len(sec) or sec[-1] == 0:
        raise ValueError("sequences bitstream missing or without its end mark")


def walk(frame: bytes) -> list[BlockInfo]:
    """Every block of a zstd frame (RFC 8878 3.1.1), with its literals and sequences section headers read."""
    frame = bytes(frame)
    if int.from_bytes(frame[:4], "little") != ZSTD_MAGIC:
        raise ValueError("not a zstd frame")
    fhd = frame[4]
    single, checksum, did = (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
    p = 5 + (not single) + (0, 1, 2, 4)[did] + ((1 if single else 0), 2, 4, 8)[fhd >> 6]
    out = []
    while True:
        h = int.from_bytes(frame[p:p + 3], "little")
        info = BlockInfo(type=(h >> 1) & 3, size=h >> 3, last=bool(h & 1))
        p += 3
        n = 1 if info.type == 1 else info.size
        body = frame[p:p + n]
        if info.type == 3 or len(body) != n:
            raise ValueError("reserved block type or truncated block")
        if info.type == 2:
            _sequences(body[_literals(body, info):], info)
        out.append(info)
        p += n
        if info.last:
            break
    if p + 4 * checksum != len(frame):
        raise ValueError("bytes after the last block")
    return out


# -- census ------------------------------------------------------------------------------------------------------------
def forms(b: BlockInfo) -> list[str]:
    """The named forms of one block."""
    out = [("block:raw", "block:rle", "block:compressed")[b.type]]
    if b.type != 2:
        return out
    if b.lit_type in (0, 1):
        out.append(f"lit:{('raw', 'rle')[b.lit_type]}/{b.lit_hdr}B")
    else:
        out.append(f"lit:{('huf', 'treeless')[b.lit_type - 2]}/sf{b.lit_sf}")
    if b.tree == "direct":
        out.append("tree:direct")
    elif b.tree == "fse":
        out.append(f"tree:fse/log{b.tree_log}/{('even', 'odd')[b.tree_weights % 2]}")
    if b.huf_maxlen == HUF_MAXBITS:
        out.append("huf:maxlen11")
    out.append("nseq:0" if b.nseq == 0 else f"nseq:{b.nseq_bytes}B")
    if b.nseq in EDGE_COUNTS:
        out.append(EDGE_COUNTS[b.nseq])
    if b.modes:
        out.append("modes:" + "".join(MODE_LETTER[m] for m in b.modes))
        out += [f"{name}:log{log}" for (name, _), log in zip(COLUMNS, b.logs) if log is not None]
    return out


def census(frames) -> Counter:
    c = Counter()
    for fr in frames:
        for b in walk(fr):
            c.update(forms(b))
    return c


_COMMON = {"block:raw", "block:rle", "block:compressed", "lit:raw/2B", "lit:raw/3B", "nseq:1B", "nseq:2B", "nseq:3B",
           *EDGE_COUNTS.values(), "modes:PPP"}
_ENTROPY = _COMMON | {"lit:huf/sf0", "lit:huf/sf2", "lit:huf/sf3", "tree:direct", "huf:maxlen11", "nseq:0",
                      "modes:RRR", "modes:RFF", "modes:FFF", "modes:FFR", "modes:FRF",
                      "LL:log5", "LL:log9", "OF:log5", "OF:log8", "ML:log5", "ML:log9"}
REQUIRED = {
    "lz": _COMMON,
    "lze": _ENTROPY,
    "lzh": _ENTROPY | {"tree:fse/log5/odd", "tree:fse/log5/even", "tree:fse/log6/odd", "tree:fse/log6/even"},
}

# Forms the encoders never write, and why.  The greedy parse (zstd_lz_ref.lz_parse) makes every byte value's first
# occurrence in a block a literal and looks matches up only in earlier 256-byte tiles.
UNREACHABLE = {
    "lit:rle/*": "a block that is not constant has >= 2 byte values, and the first occurrence of each is a literal",
    "lit:raw/1B": "a block with a sequence has its first 256-byte tile as literals; a block of <= 31 bytes has no "
                  "sequence, and its raw literals plus headers are larger than the block, so it stays a Raw_Block",
    "lit:huf/sf1": "four streams are written only when the regenerated or compressed size exceeds 1023, which sf1's "
                   "10-bit fields cannot hold",
    "lit:treeless/*": "every Huffman-coded block states its own tree",
    "nseq:0 in lz": "without sequences the _lz content is raw literals plus 2 header bytes, larger than the block",
    "modes:X": "no block refers to the previous block's tables (Repeat_Mode)",
    "modes with P beside R or F": "a block uses the predefined tables for all three columns (_lz) or for none",
    "tree:* in lz / tree:fse in lze": "_lz keeps literals raw; _lze writes the direct tree form only",
}


# -- inputs that reach the rare forms ------------------------------------------------------------------------------------
B = 128 << 10


def word_block(n_words: int = B // 4, vocab: int = 16, seed: int = 16) -> np.ndarray:
    """`vocab` words of 4 distinct bytes (4 * vocab distinct values in all); each next word drawn at random among those
    that did not follow the current word in the last 160 words.  After the first 256-byte tile, which has no earlier tile
    to match against, every word is one 4-byte match: 16 words fill a 128 KiB block with 32 704 sequences, all with
    Match_Length 4 (ML in RLE_Mode, LL and OF in FSE_Compressed_Mode).  Prefixes give any smaller count."""
    rng = np.random.default_rng(seed)
    words = rng.permutation(256)[:4 * vocab].reshape(vocab, 4).astype(np.uint8)
    seq, succ = [0], {}
    while len(seq) < n_words:
        w, t = seq[-1], len(seq) - 1
        recent = succ.setdefault(w, [])
        bad = {nx for (tt, nx) in recent if t - tt <= 160}
        nxt = int(rng.choice([x for x in range(vocab) if x not in bad]))
        recent.append((t, nxt))
        seq.append(nxt)
    return words[np.array(seq)].reshape(-1)


def mutated_period(n: int = B, period: int = 600, seed: int = 60) -> np.ndarray:
    """Each `period` bytes repeat the previous ones but for runs of 1-24 fresh bytes at random places: every match has
    offset `period` (OF in RLE_Mode) while literal runs and match lengths vary (LL and ML in FSE_Compressed_Mode)."""
    rng = np.random.default_rng(seed)
    out = np.empty(n + period, np.uint8)
    out[:period] = rng.integers(0, 256, period)
    for s in range(period, n, period):
        out[s:s + period] = out[s - period:s]
        k = int(rng.integers(2, 6))
        for p in rng.choice(period - 24, k, replace=False):
            ln = int(rng.integers(1, 25))
            out[s + p:s + p + ln] = rng.integers(0, 256, ln)
    return out[:n]


def long_literal_runs(n: int = B, seed: int = 70) -> np.ndarray:
    """Runs of 256-399 random bytes, each followed by a copy of a random stretch of it that starts in an earlier tile
    than the copy (the stretch is the copy's only earlier match): every literal length lies in [256, 511], one
    Literals_Length code (LL in RLE_Mode), while offsets and match lengths vary (OF and ML in FSE_Compressed_Mode)."""
    rng = np.random.default_rng(seed)
    out = np.empty(n + 1024, np.uint8)
    pos = 0
    while pos < n:
        r = int(rng.integers(256, 400))
        out[pos:pos + r] = rng.integers(0, 256, r)
        s, pos = pos, pos + r
        j = int(rng.integers(s, min(pos // 256 * 256, pos - 4)))
        ln = int(rng.integers(4, pos - j + 1))
        out[pos:pos + ln] = out[j:j + ln]
        pos += ln
    return out[:n]


def fib_symbols(n: int = B, nfib: int = 16, seed: int = 80) -> np.ndarray:
    """Values 64..64+nfib-1 occurring 1, 1, 2, 3, 5, ... times (Fibonacci numbers) among uniform bytes 0..63, shuffled.
    Few 4-byte keys repeat, so nearly every byte is a literal: more than 16 383 literals, all <= 128, that Huffman
    coding shrinks by a quarter (Size_Format 11 in _lze), and whose unlimited Huffman code is longer than 11 bits for
    the chain of Fibonacci counts (the length limit's halving loop runs)."""
    fib = [1, 1]
    while len(fib) < nfib:
        fib.append(fib[-1] + fib[-2])
    rng = np.random.default_rng(seed)
    rare = np.repeat(np.arange(64, 64 + nfib), fib)
    return rng.permutation(np.concatenate([rare, rng.integers(0, 64, n - len(rare))])).astype(np.uint8)


MODES = ("lz", "lze", "lzh")
_ALL, _ENT = MODES, ("lze", "lzh")


@lru_cache(maxsize=1)
def form_cases():
    """Seeded chunks that reach the forms the other GPU inputs miss -> [(chunk, {mode: forms its frame must show})].
    Built once per process; the chunks are shared, not to be written."""
    text = text_corpus(B, 81)
    words = word_block()

    def case(part, modes, *names):
        return part, {m: set(names) for m in modes}

    ent = {"nseq:3B", "modes:FFR", "LL:log9", "OF:log8"}
    out = [
        (words, {"lz": {"nseq:3B"}, "lze": ent, "lzh": ent}),                          # 32 704 sequences
        case(words[:256 + 4 * 0x7F00], _ALL, "nseq:0x7F00"),                            # the smallest 3-byte count
        case(words[:256 + 4 * 0x7EFF], _ALL, "nseq:0x7EFF"),                            # the largest 2-byte count
        case(words[:256 + 4 * 127], _ALL, "nseq:127"),
        case(words[:256 + 4 * 128], _ALL, "nseq:128"),
        case(np.random.default_rng(82).choice(np.array([3, 9], np.uint8), 259), _ENT, "nseq:0", "lit:huf/sf0"),
        case(mutated_period(), _ENT, "modes:FRF"),
        case(long_literal_runs(), _ENT, "modes:RFF"),
        case(fib_symbols(), _ENT, "huf:maxlen11", "lit:huf/sf3"),
        case(text[:900], _ENT, "LL:log5", "OF:log5", "ML:log5"),                        # < 128 sequences
    ]
    for top in (124, 125, 200, 201):                                                     # FSE tree, weight log 5 / 6
        t = text.copy()
        t[::991] = top
        out.append(case(t, ("lzh",), f"tree:fse/log{5 if top < 128 else 6}/{('even', 'odd')[top % 2]}"))
    return out


def form_parts() -> list[np.ndarray]:
    return [p for p, _ in form_cases()]
