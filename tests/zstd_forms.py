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


# -- a decoder that names the edges it passes ----------------------------------------------------------------------------
# decode_payload() reads a blob payload (zstd and skippable frames) as RFC 8878 describes it, with upstream's window
# limit, and counts in `forms` every edge of the format it passes.  It is the census of tests/zstd_edge_frames.py: the
# forms are read from the bytes, not claimed by the builder.  Edge names:
#   rep:1 .. rep:3 | rep:1/ll0 .. rep:3/ll0     a repeat offset code with Literals_Length > 0 / == 0 (rep:3/ll0: rep0 - 1)
#   rep:3/ll0/twice                            rep0 - 1 in two sequences in a row
#   rep:across-block | rep:across-raw | rep:reset   a repeat code before any new offset in a block: the history from an
#                                              earlier block, from before a Raw block, or the reset one of a later frame
#   off:<k>/overlap (k <= 33) | off:overlap   a match at least 32 bytes longer than its offset k; longer than it
#   off:all | off:into-raw | off:into-rle      offset == the bytes so far of a frame after the first; a match that starts
#                                              in an earlier Raw / RLE block and runs past its end
#   off:raw-to-rle                             such a match that runs from a Raw block into the RLE block after it
#   ll:code35 | ml:code52 | of:code<k>        codes (OF from 20 on)
#   seq:wide/ll<b>/ml<b>                       a sequence with >= 15 LL, >= 15 ML and >= 23 OF extra bits
#   logs:<ll>/<of>/<ml>                        the accuracy logs of a block whose three tables are FSE_Compressed
#   <col>:log<k> | <col>:rle/max | <col>:maxsym | <col>:X-after-<P|R|F>   a table's accuracy log, its largest code in
#                                              RLE_Mode or an FSE description, Repeat_Mode after each mode
#   fse:less1 | fse:zeros+3 | fse:zeros+4+    a "less than 1" count; a zero count with exactly 3 / more than 3 more
#   lit:<form>:max                             the largest size of a literals header form (raw/1B .. 3B, huf/sf0 .. sf3)
#   huf:last0 | huf:last1 | huf4:n<6..9>      four streams whose last one holds 0 / 1 symbols; of 6..9 literals
#   lit:treeless/1x | lit:treeless/4x | huf:maxbits11 | huf:256sym | tree:direct/128   Huffman literals
#   window:m<0..7> | block:bmax/<raw|rle|compressed> | block:content-128k   Window_Descriptor mantissas; blocks of
#                                              Block_Maximum_Size under a smaller window; a 128 KiB Compressed_Block content
#   fcs:2/256 | fcs:2/65791 | frame:empty | checksum:unaligned
#   reject:<rule>                              the rule a payload breaks (decode_payload raises Reject)
LL_MAXLOG, OF_MAXLOG, ML_MAXLOG = 9, 8, 9
HUF_MAXLOG = 11
WINDOW_MAX = (1 << 27) + 1        # libzstd's default: windowLogMax 27, a Window_Size of at most 2^27 + 1 bytes
BLOCK_MAX = 128 << 10


class Reject(ValueError):
    """A payload that breaks a rule of the format; `rule` names it."""

    def __init__(self, rule: str):
        super().__init__(rule)
        self.rule = rule


class _Back:
    """Backward bitstream (RFC 8878 4.1): the highest set bit of the last byte marks its end.  `bit` counts the bits not
    read yet; reads past the start give zeros and drive it negative."""

    def __init__(self, data: bytes, what: str):
        if not data or data[-1] == 0:
            raise Reject(f"{what}:end-mark")
        self.v = int.from_bytes(data, "little")
        self.bit = 8 * (len(data) - 1) + data[-1].bit_length() - 1

    def peek(self, n: int) -> int:
        lo = self.bit - n
        return ((self.v >> lo) if lo >= 0 else (self.v << -lo)) & ((1 << n) - 1)

    def read(self, n: int) -> int:
        v = self.peek(n)
        self.bit -= n
        return v

    def end(self, what: str):
        if self.bit:
            raise Reject(f"{what}:bits-{'left' if self.bit > 0 else 'missing'}")


def xxh64(data: bytes, seed: int = 0) -> int:
    """XXH64 of `data` (the frame content checksum is its low 32 bits)."""
    P1, P2, P3, P4, P5 = (0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63,
                          0x27D4EB2F165667C5)
    M = (1 << 64) - 1

    def rotl(x, r):
        return ((x << r) | (x >> (64 - r))) & M

    def rnd(acc, v):
        return rotl((acc + v * P2) & M, 31) * P1 & M

    n, i = len(data), 0
    if n >= 32:
        v = [(seed + P1 + P2) & M, (seed + P2) & M, seed, (seed - P1) & M]
        w = np.frombuffer(data[:n // 32 * 32], "<u8").reshape(-1, 4).tolist()
        for row in w:
            v = [rnd(v[k], row[k]) for k in range(4)]
        i = n // 32 * 32
        h = (rotl(v[0], 1) + rotl(v[1], 7) + rotl(v[2], 12) + rotl(v[3], 18)) & M
        for x in v:
            h = ((h ^ rnd(0, x)) * P1 + P4) & M
    else:
        h = (seed + P5) & M
    h = (h + n) & M
    while i + 8 <= n:
        h = (rotl(h ^ rnd(0, int.from_bytes(data[i:i + 8], "little")), 27) * P1 + P4) & M
        i += 8
    if i + 4 <= n:
        h = (rotl(h ^ (int.from_bytes(data[i:i + 4], "little") * P1 & M), 23) * P2 + P3) & M
        i += 4
    while i < n:
        h = rotl(h ^ (data[i] * P5 & M), 11) * P1 & M
        i += 1
    h ^= h >> 33
    h = h * P2 & M
    h ^= h >> 29
    h = h * P3 & M
    return h ^ (h >> 32)


def huf_weights(body: bytes):
    """A Huffman_Tree_Description at body[0:] -> (its size, the weights of every symbol, the implied last one included,
    the table log)."""
    th = body[0]
    if th >= 128:
        nw = th - 127
        size = 1 + (nw + 1) // 2
        if len(body) < size:
            raise Reject("tree:truncated")
        w = [(body[1 + k // 2] >> (4 if k % 2 == 0 else 0)) & 15 for k in range(nw)]
    else:
        size = 1 + th
        if len(body) < size:
            raise Reject("tree:truncated")
        try:
            log, w = fse_weights_decode(body[1:size])
        except (ValueError, IndexError):
            raise Reject("tree:weights") from None
        if log > 6 or len(w) > 255:
            raise Reject("tree:weights")
    if max(w) > HUF_MAXLOG:
        raise Reject("tree:weights")
    total = sum(1 << (x - 1) for x in w if x)
    if total == 0:
        raise Reject("tree:weights")
    log = total.bit_length()
    rest = (1 << log) - total
    if log > HUF_MAXLOG:
        raise Reject("tree:maxbits")
    if rest & (rest - 1):
        raise Reject("tree:incomplete")
    return size, w + [rest.bit_length()], log


class _Frame:
    def __init__(self):
        self.rep = [1, 4, 8]
        self.huf = None                   # (decoding table, log) of the last tree
        self.tab = [None, None, None]     # (decoding table, log, mode it was built in) per column
        self.spans = []                   # (start, end, block type) of the frame's Raw and RLE blocks


def _huf_table(w, log):
    table = []
    for wt in range(1, log + 1):
        for s, x in enumerate(w):
            if x == wt:
                table += [(s, log + 1 - wt)] * (1 << (wt - 1))
    return table


def _huf_stream(data: bytes, table, log, n: int, what: str = "huf") -> bytes:
    r = _Back(data, what)
    out = bytearray(n)
    for k in range(n):
        s, nb = table[r.peek(log)]
        out[k] = s
        r.bit -= nb
    r.end(what)
    return bytes(out)


_LIT_MAX = {("raw", 1): 31, ("raw", 2): 4095, ("huf", 0): 1023, ("huf", 1): 1023, ("huf", 2): 16383}


def _decode_literals(body: bytes, f: _Frame, bmax: int, forms: Counter):
    """The Literals_Section at body[0:] -> (literals, its size)."""
    if not body:
        raise Reject("lit:truncated")
    t, sf = body[0] & 3, (body[0] >> 2) & 3
    if t < 2:
        h = 1 if sf in (0, 2) else 2 if sf == 1 else 3
        if len(body) < h:
            raise Reject("lit:truncated")
        v = int.from_bytes(body[:h], "little")
        n = v >> 3 if h == 1 else v >> 4
        if n > bmax:
            raise Reject("lit:size")
        kind = ("raw", "rle")[t]
        if n == _LIT_MAX.get(("raw", h)) or (h == 3 and n >= BLOCK_MAX - 5):
            forms[f"lit:{kind}/{h}B:max"] += 1
        if t == 0:
            if len(body) < h + n:
                raise Reject("lit:truncated")
            return body[h:h + n], h + n
        if len(body) < h + 1:
            raise Reject("lit:truncated")
        return body[h:h + 1] * n, h + 1
    h, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
    if len(body) < h:
        raise Reject("lit:truncated")
    v = int.from_bytes(body[:h], "little")
    regen, csize = (v >> 4) & ((1 << bits) - 1), (v >> (4 + bits)) & ((1 << bits) - 1)
    four = sf != 0
    if regen > bmax or h + csize > len(body):
        raise Reject("lit:size")
    if four and regen < 6:
        raise Reject("huf:4x-small")
    if regen == _LIT_MAX.get(("huf", sf)) or (sf == 3 and regen == BLOCK_MAX):
        forms[f"lit:huf/sf{sf}:max"] += 1
    q = body[h:h + csize]
    if t == 2:
        size, w, log = huf_weights(q)
        f.huf = (_huf_table(w, log), log)
        q = q[size:]
        if log == 11:
            forms["huf:maxbits11"] += 1
        if len(w) == 256:
            forms["huf:256sym"] += 1
        if body[h] == 255:
            forms["tree:direct/128"] += 1
    elif f.huf is None:
        raise Reject("lit:treeless-none")
    table, log = f.huf
    if t == 3:
        forms[f"lit:treeless/{'4x' if four else '1x'}"] += 1
    if four and regen <= 9:
        forms[f"huf4:n{regen}"] += 1
    if not four:
        return _huf_stream(q, table, log, regen), h + csize
    if len(q) < 6:
        raise Reject("lit:size")
    l1, l2, l3 = (int.from_bytes(q[k:k + 2], "little") for k in (0, 2, 4))
    if l1 + l2 + l3 > len(q) - 6:
        raise Reject("lit:size")
    seg = (regen + 3) // 4
    cuts = [6, 6 + l1, 6 + l1 + l2, 6 + l1 + l2 + l3, len(q)]
    lits = b"".join(_huf_stream(q[cuts[k]:cuts[k + 1]], table, log, seg if k < 3 else regen - 3 * seg, f"huf4:s{k}")
                    for k in range(4))
    if regen - 3 * seg <= 1:
        forms[f"huf:last{regen - 3 * seg}"] += 1
    return lits, h + csize


_COL_MAXLOG = (LL_MAXLOG, OF_MAXLOG, ML_MAXLOG)
_PREDEF = {}


def _decode_table(sec: bytes, pos: int, c: int, mode: int, f: _Frame, forms: Counter) -> int:
    name, maxsym = COLUMNS[c]
    if mode == 3:
        if f.tab[c] is None:
            raise Reject("modes:repeat-none")
        forms[f"{name}:X-after-{MODE_LETTER[f.tab[c][2]]}"] += 1
        return pos
    if mode == 0:
        if not _PREDEF:
            from zstd_lz_ref import LL_NORM, OF_NORM, ML_NORM
            for k, (norm, log) in enumerate(((LL_NORM, 6), (OF_NORM, 5), (ML_NORM, 6))):
                _PREDEF[k] = (fse_decoding_table(norm, log), log)
        f.tab[c] = (*_PREDEF[c], 0)
        return pos
    if mode == 1:
        if pos >= len(sec) or sec[pos] > maxsym:
            raise Reject("table:rle-symbol")
        if sec[pos] == (24 if c == 1 else maxsym):      # OF: 24, the largest code a 16 MiB chunk can use
            forms[f"{name}:rle/max"] += 1
        f.tab[c] = ([(sec[pos], 0, 0)], 0, 1)
        return pos + 1
    if pos >= len(sec):
        raise Reject("table:description")
    if (sec[pos] & 15) + 5 > _COL_MAXLOG[c]:
        raise Reject("table:log")
    try:
        log, counts, end = read_fse_description(sec + bytes(8), pos, maxsym)
    except (ValueError, IndexError):
        raise Reject("table:description") from None
    if end > len(sec):
        raise Reject("table:description")
    forms[f"{name}:log{log}"] += 1
    if len(counts) == maxsym + 1:
        forms[f"{name}:maxsym"] += 1
    if -1 in counts:
        forms["fse:less1"] += 1
    run = 0
    for x in counts + [1]:
        if x == 0:
            run += 1
            continue
        if run == 4:
            forms["fse:zeros+3"] += 1
        elif run > 4:
            forms["fse:zeros+4+"] += 1
        run = 0
    f.tab[c] = (fse_decoding_table(counts, log), log, 2)
    return end


def _decode_block(body: bytes, f: _Frame, out: bytearray, fstart: int, bmax: int, first_seq_block: bool,
                  after_raw: bool, later_frame: bool, forms: Counter) -> bool:
    """A Compressed_Block's content appended to out; True when it has sequences."""
    from zstd_lz_ref import LL_BASE, LL_BITS, ML_BASE, ML_BITS
    lits, used = _decode_literals(body, f, bmax, forms)
    sec = body[used:]
    if not sec:
        raise Reject("seq:truncated")
    n, k = sec[0], 1
    if n == 0:
        if len(sec) != 1:
            raise Reject("seq:trailing")
    elif n == 255:
        if len(sec) < 3:
            raise Reject("seq:truncated")
        n, k = sec[1] + (sec[2] << 8) + 0x7F00, 3
    elif n >= 128:
        if len(sec) < 2:
            raise Reject("seq:truncated")
        n, k = ((n - 128) << 8) + sec[1], 2
    b0, lpos = len(out), 0
    if n:
        if k >= len(sec):
            raise Reject("seq:truncated")
        m = sec[k]
        if m & 3:
            raise Reject("modes:reserved")
        pos = k + 1
        for c in range(3):
            pos = _decode_table(sec, pos, c, (m >> (6 - 2 * c)) & 3, f, forms)
        r = _Back(sec[pos:], "seq")
        (tl, gl, _), (to, go, _), (tm, gm, _) = f.tab
        if (m >> 2) & 0x3F == 0b101010:
            forms[f"logs:{gl}/{go}/{gm}"] += 1
        sl, so, sm = r.read(gl), r.read(go), r.read(gm)
        new_offset, prev_idx = False, -1
        for j in range(n):
            lc, lb, lbase = tl[sl]
            oc, ob, obase = to[so]
            mc, mb, mbase = tm[sm]
            ov = (1 << oc) + r.read(oc)
            ml = ML_BASE[mc] + r.read(ML_BITS[mc])
            ll = LL_BASE[lc] + r.read(LL_BITS[lc])
            if j + 1 < n:
                sl, sm, so = lbase + r.read(lb), mbase + r.read(mb), obase + r.read(ob)
            rep = f.rep
            if ov > 3:
                off = ov - 3
                f.rep = [off, rep[0], rep[1]]
                new_offset, prev_idx = True, -1
            else:
                idx = ov - 1 + (ll == 0)
                forms[f"rep:{ov}" + ("/ll0" if ll == 0 else "")] += 1
                if idx == 3 and prev_idx == 3:
                    forms["rep:3/ll0/twice"] += 1
                prev_idx = idx
                if not new_offset:
                    if later_frame and first_seq_block:
                        forms["rep:reset"] += 1
                    elif not first_seq_block:
                        forms["rep:across-raw" if after_raw else "rep:across-block"] += 1
                off = (rep[0], rep[1], rep[2], rep[0] - 1)[idx]
                f.rep = ([rep[0], rep[1], rep[2]], [rep[1], rep[0], rep[2]], [rep[2], rep[0], rep[1]],
                         [rep[0] - 1, rep[0], rep[1]])[idx]
            if lpos + ll > len(lits):
                raise Reject("seq:literals-overrun")
            if len(out) + ll + ml - b0 > bmax:
                raise Reject("block:decoded-size")
            here = len(out) + ll
            if off <= 0:
                raise Reject("seq:offset-zero")
            if off > here - fstart:
                raise Reject("seq:offset-beyond")
            forms[f"ll:code{lc}"] += lc == 35
            forms[f"ml:code{mc}"] += mc == 52
            forms[f"of:code{oc}"] += oc >= 20
            if LL_BITS[lc] >= 15 and ML_BITS[mc] >= 15 and oc >= 23:
                forms[f"seq:wide/ll{LL_BITS[lc]}/ml{ML_BITS[mc]}"] += 1
            if off == here - fstart and fstart:
                forms["off:all"] += 1
            for i, (s0, s1, bt) in enumerate(f.spans):
                if s0 <= here - off < s1 < here - off + ml:
                    forms[f"off:into-{bt}"] += 1
                    if i + 1 < len(f.spans) and f.spans[i + 1][0] == s1:
                        forms[f"off:{bt}-to-{f.spans[i + 1][2]}"] += 1
            out += lits[lpos:lpos + ll]
            lpos += ll
            if off < ml:
                forms["off:overlap"] += 1
                if off <= 33 and ml >= off + 32:
                    forms[f"off:{off}/overlap"] += 1
                src = out[here - off:here]
                out += (src * (ml // off + 1))[:ml]
            else:
                out += out[here - off:here - off + ml]
        r.end("seq")
    if len(out) + len(lits) - lpos - b0 > bmax:
        raise Reject("block:decoded-size")
    out += lits[lpos:]
    return n > 0


def decode_payload(payload: bytes, forms: Counter | None = None) -> bytes:
    """The content of a blob payload: zstd frames with skippable frames between them.  Raises Reject; counts the edges
    it passes in `forms`."""
    forms = Counter() if forms is None else forms
    data, out, q, nframe = bytes(payload), bytearray(), 0, 0
    while q < len(data):
        if len(data) - q < 4:
            raise Reject("frame:truncated")
        magic = int.from_bytes(data[q:q + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            if len(data) - q < 8:
                raise Reject("skippable:header")
            if int.from_bytes(data[q + 4:q + 8], "little") > len(data) - q - 8:
                raise Reject("skippable:truncated")
            q += 8 + int.from_bytes(data[q + 4:q + 8], "little")
            continue
        if magic != ZSTD_MAGIC:
            raise Reject("frame:magic")
        q += 4
        if q >= len(data):
            raise Reject("frame:truncated")
        fhd = data[q]
        q += 1
        single, checksum, did = (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
        if fhd & 8:
            raise Reject("frame:reserved")
        window = 0
        if not single:
            if q >= len(data):
                raise Reject("frame:truncated")
            wd = data[q]
            q += 1
            wlog = 10 + (wd >> 3)
            window = (1 << wlog) + ((1 << wlog) >> 3) * (wd & 7)
        dsz, fsz = (0, 1, 2, 4)[did], ((1 if single else 0), 2, 4, 8)[fhd >> 6]
        if len(data) - q < dsz + fsz:
            raise Reject("frame:truncated")
        if any(data[q:q + dsz]):
            raise Reject("frame:dictionary")
        q += dsz
        fcs = int.from_bytes(data[q:q + fsz], "little") + (256 if fsz == 2 else 0)
        q += fsz
        if fsz == 2 and fcs in (256, 65791):
            forms[f"fcs:2/{fcs}"] += 1
        if single:
            window = fcs
        if window > WINDOW_MAX:
            raise Reject("frame:window/" + ("single" if single else f"m{wd & 7}"))
        if not single:
            forms[f"window:m{wd & 7}"] += 1
        bmax = min(window, BLOCK_MAX)
        f, fstart = _Frame(), len(out)
        seq_blocks, prev_raw = 0, False
        while True:
            if len(data) - q < 3:
                raise Reject("frame:truncated")
            bh = int.from_bytes(data[q:q + 3], "little")
            q += 3
            bt, bsize = (bh >> 1) & 3, bh >> 3
            start = len(out)
            if bt == 3:
                raise Reject("block:reserved")
            if bt == 0:
                if bsize > bmax:
                    raise Reject("block:size/raw")
                if bsize > len(data) - q:
                    raise Reject("frame:truncated")
                out += data[q:q + bsize]
                q += bsize
            elif bt == 1:
                if bsize > bmax:
                    raise Reject("block:size/rle")
                if q >= len(data):
                    raise Reject("frame:truncated")
                out += data[q:q + 1] * bsize
                q += 1
            else:
                if bsize == BLOCK_MAX:
                    forms["block:content-128k"] += 1
                if bsize > bmax:
                    raise Reject("block:size/compressed")
                if bsize > len(data) - q:
                    raise Reject("frame:truncated")
                if _decode_block(data[q:q + bsize], f, out, fstart, bmax, seq_blocks == 0, prev_raw, nframe > 0,
                                 forms):
                    seq_blocks += 1
                q += bsize
            kind = ("raw", "rle", "compressed")[bt]
            if bt < 2:
                f.spans.append((start, len(out), kind))
            prev_raw = bt == 0 and seq_blocks > 0
            if not single and len(out) - start == bmax and bmax < BLOCK_MAX:
                forms[f"block:bmax/{kind}"] += 1
            if bh & 1:
                break
        if fsz and len(out) - fstart != fcs:
            raise Reject("frame:content-size")
        if len(out) == fstart:
            forms["frame:empty"] += 1
        if checksum:
            if len(data) - q < 4:
                raise Reject("frame:truncated")
            if xxh64(bytes(out[fstart:])) & 0xFFFFFFFF != int.from_bytes(data[q:q + 4], "little"):
                raise Reject("frame:checksum")
            if fstart % 8 and len(out) - fstart >= 32:
                forms["checksum:unaligned"] += 1
            q += 4
        nframe += 1
    return bytes(out)


# The edges tests/zstd_edge_frames.edge_cases() must reach, read by decode_payload (tests/test_zstd_edges_cpu.py checks
# the set, and that every case reaches one of them that no other case reaches; the GPU tests decode every case)
REQUIRED_EDGES = {
    "rep:1", "rep:2", "rep:3", "rep:1/ll0", "rep:2/ll0", "rep:3/ll0", "rep:3/ll0/twice",
    "rep:across-block", "rep:across-raw", "rep:reset",
    *(f"off:{k}/overlap" for k in range(1, 34)), "off:overlap", "off:all", "off:into-raw", "off:into-rle",
    "off:raw-to-rle",
    "ll:code35", "ml:code52", "of:code24", "seq:wide/ll16/ml15", "seq:wide/ll15/ml16",
    *(f"{c}:log{k}" for c in ("LL", "ML") for k in range(5, 10)), *(f"OF:log{k}" for k in range(5, 9)),
    "logs:5/5/5", "logs:6/6/6", "logs:7/7/7", "logs:8/8/8", "logs:9/8/9",
    "LL:rle/max", "OF:rle/max", "ML:rle/max", "LL:maxsym", "OF:maxsym", "ML:maxsym",
    "fse:less1", "fse:zeros+3", "fse:zeros+4+",
    "LL:X-after-P", "LL:X-after-F", "OF:X-after-P", "OF:X-after-R", "ML:X-after-R", "ML:X-after-F",
    "lit:raw/1B:max", "lit:raw/2B:max", "lit:raw/3B:max", "lit:rle/3B:max",
    "lit:huf/sf0:max", "lit:huf/sf1:max", "lit:huf/sf2:max", "lit:huf/sf3:max",
    "huf:last0", "huf:last1", "huf4:n6", "huf4:n7", "huf4:n8", "huf4:n9", "lit:treeless/1x", "lit:treeless/4x",
    "huf:maxbits11", "huf:256sym", "tree:direct/128",
    *(f"window:m{k}" for k in range(8)), "block:bmax/raw", "block:bmax/rle", "block:bmax/compressed",
    "block:content-128k", "fcs:2/256", "fcs:2/65791", "frame:empty", "checksum:unaligned",
    # rejections: K13's rules (DESIGN.md K13) and the stream ends
    "reject:frame:window/m0", "reject:frame:window/m1", "reject:frame:window/single", "reject:frame:reserved",
    "reject:frame:dictionary", "reject:block:reserved", "reject:block:size/raw", "reject:block:size/rle",
    "reject:block:size/compressed", "reject:block:decoded-size", "reject:frame:content-size", "reject:frame:checksum",
    "reject:frame:magic", "reject:skippable:header", "reject:skippable:truncated",
    "reject:seq:offset-zero", "reject:seq:offset-beyond", "reject:seq:literals-overrun", "reject:seq:trailing",
    "reject:modes:repeat-none", "reject:modes:reserved", "reject:table:rle-symbol", "reject:table:log",
    "reject:table:description", "reject:seq:bits-left", "reject:seq:bits-missing", "reject:seq:end-mark",
    "reject:lit:treeless-none", "reject:lit:size", "reject:huf:4x-small", "reject:huf:bits-left", "reject:huf:bits-missing",
    *(f"reject:huf4:s{k}:bits-{e}" for k in range(4) for e in ("left", "missing")), "reject:huf:end-mark",
    "reject:tree:incomplete", "reject:tree:weights",
}
