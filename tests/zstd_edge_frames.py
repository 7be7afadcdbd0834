"""Hand-built zstd payloads at the edges of RFC 8878, for the blob decoder (K13, csrc/zdec.cu).  Test infrastructure for
tests/test_zstd_edges_cpu.py and tests/test_gpu_zstd_edges.py.

A frame is built from an explicit spec: the frame header fields; per block its type, and for a Compressed_Block the
literals form (Raw, RLE, Huffman with the code lengths and the tree form, or Treeless; 1 or 4 streams; the header's
Size_Format) and the sequences as raw (Literals_Length, Offset_Value, Match_Length), so the repeat codes 1 to 3 can be
written, with each column's table mode and normalized counts.  The writers are the restatements' own: zstd_ent_ref's
bit writer, FSE table description, Huffman codes, streams and sequence bitstream, zstd_huf_ref's FSE-compressed
weights, zstd_lz_ref's code tables.

edge_cases() builds every case when the tests run, so no binary fixture is needed.  The content of a valid case is what
zstd_forms.decode_payload (the RFC decoder) reads from it; tests/test_zstd_edges_cpu.py checks that libzstd's streaming
decoder reads the same bytes, and refuses every invalid case.  Which edges the cases reach is measured from the bytes by
decode_payload and checked against zstd_forms.REQUIRED_EDGES."""
from __future__ import annotations

from functools import lru_cache
from typing import NamedTuple

import numpy as np

import zstd_forms as zf
from pbs_plus_b200 import _lib
from zstd_ent_ref import _Bits, fse_description, huf_codes, huf_stream, seq_bitstream_tables
from zstd_huf_ref import fse_weights
from zstd_lz_ref import LL_LOG, LL_NORM, ML_LOG, ML_NORM, OF_LOG, OF_NORM, fse_table, seq_codes

MAGIC = b"\x28\xb5\x2f\xfd"


class Case(NamedTuple):
    name: str
    payload: bytes
    content: bytes | None        # None: the payload is invalid
    status: int                  # the DEC_* status K13 must give
    size: int                    # the chunk_len to decode it with


# -- frames and blocks ---------------------------------------------------------------------------------------------------
def raw(data: bytes):
    return (0, len(data), bytes(data))


def rle(byte: int, n: int):
    return (1, n, bytes([byte]))


def comp(body: bytes):
    return (2, len(body), body)


def frame(blocks, fcs: int | None = None, single: bool = False, wd: int = 0x58, checksum: bytes | None = None,
          fcs_size: int | None = None, fhd_or: int = 0, did: bytes = b"") -> bytes:
    """A frame of the blocks (the last one gets Last_Block).  fcs: Frame_Content_Size (None: absent; the field takes the
    smallest size that holds it unless fcs_size says); single: Single_Segment (no Window_Descriptor), else `wd`;
    checksum: the content, whose XXH64 is appended; fhd_or: bits or-ed into the descriptor; did: a Dictionary_ID field."""
    if fcs is None:
        size = 0
    else:
        size = fcs_size or (1 if single and fcs < 256 else 2 if 256 <= fcs <= 65791 else 4 if fcs < 1 << 32 else 8)
    flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[size]
    fhd = flag << 6 | single << 5 | (checksum is not None) << 2 | {0: 0, 1: 1, 2: 2, 4: 3}[len(did)] | fhd_or
    out = bytearray(MAGIC + bytes([fhd]))
    if not single:
        out.append(wd)
    out += did
    if size:
        out += (fcs - 256 if size == 2 else fcs).to_bytes(size, "little")
    for k, (t, n, body) in enumerate(blocks):
        out += ((k + 1 == len(blocks)) | t << 1 | n << 3).to_bytes(3, "little") + body
    if checksum is not None:
        out += (zf.xxh64(bytes(checksum)) & 0xFFFFFFFF).to_bytes(4, "little")
    return bytes(out)


def skippable(n: int, fill: int = 0x5A) -> bytes:
    return (0x184D2A53).to_bytes(4, "little") + n.to_bytes(4, "little") + bytes([fill]) * n


# -- literals ------------------------------------------------------------------------------------------------------------
def lit_raw(data: bytes, h: int | None = None) -> bytes:
    n = len(data)
    h = h or (1 if n <= 31 else 2 if n <= 4095 else 3)
    hdr = bytes([n << 3]) if h == 1 else (0b0100 | n << 4).to_bytes(2, "little") if h == 2 else \
        (0b1100 | n << 4).to_bytes(3, "little")
    return hdr + bytes(data)


def lit_rle(byte: int, n: int) -> bytes:
    h = 1 if n <= 31 else 2 if n <= 4095 else 3
    hdr = bytes([1 | n << 3]) if h == 1 else (1 | 0b0100 | n << 4).to_bytes(2, "little") if h == 2 else \
        (1 | 0b1100 | n << 4).to_bytes(3, "little")
    return hdr + bytes([byte])


def tree(lengths, form: str) -> bytes:
    """Huffman_Tree_Description of the code lengths (256 entries, 0 = absent): "direct" (4-bit weights) or "fse"."""
    mx, top = max(lengths), max(s for s in range(256) if lengths[s])
    wts = [mx + 1 - lengths[s] if lengths[s] else 0 for s in range(top)]
    if form == "direct":
        w2 = wts + [0]
        return bytes([127 + top]) + bytes(w2[k] << 4 | w2[k + 1] for k in range(0, top, 2))
    body = fse_weights(wts)
    assert body is not None and len(body) < 128
    return bytes([len(body)]) + body


def shift(stream: bytes, by: int) -> bytes:
    """A backward bitstream with one bit added below its first bit (by = 1: one left over) or its first bit dropped
    (by = -1: one missing)."""
    v = int.from_bytes(stream, "little")
    v = v << 1 if by > 0 else v >> 1
    return v.to_bytes((v.bit_length() + 7) // 8, "little")


def lit_huf(data: bytes, lengths, form: str | None = "direct", streams: int = 1, sf: int | None = None,
            tweak=None) -> bytes:
    """Compressed_Literals_Block (form "direct" / "fse": the tree stated) or Treeless_Literals_Block (form None: the
    previous tree's lengths).  tweak(k, stream) may alter stream k."""
    a = np.frombuffer(bytes(data), np.uint8)
    codes, ln = np.array(huf_codes(lengths), np.int64), np.array(lengths, np.int64)
    n = len(a)
    if streams == 1:
        parts = [huf_stream(a, codes, ln)]
    else:
        seg = (n + 3) // 4
        parts = [huf_stream(a[k * seg:min(n, (k + 1) * seg)], codes, ln) for k in range(4)]
    if tweak:
        parts = [tweak(k, p) for k, p in enumerate(parts)]
    body = (tree(lengths, form) if form else b"")
    if streams == 4:
        body += b"".join(len(p).to_bytes(2, "little") for p in parts[:3])
    body += b"".join(parts)
    c = len(body)
    if sf is None:
        sf = 0 if streams == 1 else 1 if max(n, c) <= 1023 else 2 if max(n, c) <= 16383 else 3
    t = 2 if form else 3
    h, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
    return (t | sf << 2 | n << 4 | c << (4 + bits)).to_bytes(h, "little") + body


def lengths_of(spec: dict[int, int]) -> list[int]:
    out = [0] * 256
    for s, ln in spec.items():
        out[s] = ln
    return out


# -- sequences -----------------------------------------------------------------------------------------------------------
_PRE = {0: (LL_NORM, LL_LOG), 1: (OF_NORM, OF_LOG), 2: (ML_NORM, ML_LOG)}
NSYM = (36, 32, 53)


def _table(c: int, spec):
    """(mode, description, fse_table, log) of column c: ("P",), ("R", code), ("F", norm, log) or ("X", inner spec)."""
    kind = spec[0]
    if kind == "P":
        norm, log = _PRE[c]
        return 0, b"", fse_table(norm, log), log
    if kind == "R":
        norm = [0] * NSYM[c]
        norm[spec[1]] = 1
        return 1, bytes([spec[1]]), fse_table(norm, 0), 0
    if kind == "F":
        return 2, fse_description(spec[1], spec[2]), fse_table(spec[1], spec[2]), spec[2]
    _, _, tab, log = _table(c, spec[1])
    return 3, b"", tab, log


def seq_section(seqs, ll=("P",), of=("P",), ml=("P",), tweak=None, modes_or: int = 0) -> bytes:
    """Sequences_Section of (Literals_Length, Offset_Value, Match_Length) triples with the given column tables.
    tweak(stream) may alter the bitstream."""
    n = len(seqs)
    if n == 0:
        return b"\0"
    cnt = bytes([n]) if n < 128 else bytes([(n >> 8) + 0x80, n & 0xFF]) if n < 0x7F00 else \
        b"\xff" + (n - 0x7F00).to_bytes(2, "little")
    (ml_, dl, tl, gl), (mo, do, to, go), (mm, dm, tm, gm) = _table(0, ll), _table(1, of), _table(2, ml)
    codes = [seq_codes(a, c, b - 3) for a, b, c in seqs]
    bs = seq_bitstream_tables(codes, tl, tm, to, (gl, gm, go))
    if tweak:
        bs = tweak(bs)
    return cnt + bytes([ml_ << 6 | mo << 4 | mm << 2 | modes_or]) + dl + do + dm + bs


def norm_of(codes, nsym: int, log: int) -> list[int]:
    """Counts summing to 2^log over the given codes (each at least 1), the rest on the first."""
    norm = [0] * nsym
    for c in codes:
        norm[c] = 1
    norm[codes[0]] += (1 << log) - sum(norm)
    return norm


def rand(n: int, seed: int) -> bytes:
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


# -- the cases -----------------------------------------------------------------------------------------------------------
def _valid():
    """(name, payload) of every valid case."""
    out = []
    add = lambda name, payload: out.append((name, payload))   # noqa: E731
    t = rand(4096, 1)
    # every repeat code with ll > 0 and ll == 0 (rep0 - 1 twice in a row), so every history update is read back
    add("rep_chain", frame([comp(lit_raw(t[:64]) + seq_section(
        [(20, 9 + 3, 6), (1, 20 + 3, 4), (1, 17 + 3, 5), (0, 3, 4), (0, 3, 4), (2, 2, 4), (0, 2, 5), (3, 3, 4),
         (0, 1, 6), (2, 1, 4), (5, 2, 4), (0, 3, 3)]))], None, wd=0x00))
    # the history carried across blocks, and across a Raw block
    add("rep_across_blocks", frame([comp(lit_raw(t[:32]) + seq_section([(20, 11 + 3, 6), (4, 5 + 3, 4)])),
                                    comp(lit_raw(t[32:48]) + seq_section([(3, 2, 5), (0, 2, 4), (4, 1, 4)]))],
                                   None, wd=0x00))
    add("rep_across_raw", frame([comp(lit_raw(t[:32]) + seq_section([(20, 11 + 3, 6), (4, 5 + 3, 4)])),
                                 raw(t[100:140]),
                                 comp(lit_raw(t[48:60]) + seq_section([(3, 1, 5), (0, 1, 4), (4, 3, 4)]))],
                                None, wd=0x00))
    # the history reset at the second frame: codes 1 / 2 / 3 then mean 1, 4, 8 again
    f1 = frame([comp(lit_raw(t[:40]) + seq_section([(30, 13 + 3, 6), (2, 25 + 3, 5)]))], None, wd=0x00)
    add("rep_reset", f1 + frame([comp(lit_raw(t[200:220]) + seq_section([(9, 1, 4), (1, 3, 5), (1, 2, 4), (0, 2, 4)]))],
                                None, wd=0x00))
    # every offset 1..33 with a longer match: the period copy across the 32 lanes
    for off in range(1, 34):
        ml = 3 * off + 40
        add(f"overlap{off}", frame([comp(lit_raw(t[:off + 2]) + seq_section([(off, off + 3, ml), (2, off + 3, ml + 7)]))],
                                   None, wd=0x00))
    # offset == every byte decoded so far in the frame (after a first frame, so the frame start counts)
    add("off_all", frame([raw(t[:17])], None, wd=0x00) +
        frame([comp(lit_raw(t[300:340]) + seq_section([(25, 25 + 3, 30), (5, 60 + 3, 64)]))], None, wd=0x00))
    # a match reaching back into an earlier Raw and an earlier RLE block
    add("off_into_raw_rle", frame([raw(t[400:500]), rle(0x33, 200),
                                   comp(lit_raw(t[:8]) + seq_section([(4, 210 + 3, 40), (4, 98 + 3, 60)]))],
                                  None, wd=0x00))
    # a 16 MiB chunk's largest OF code (24), and sequences with 16 + 15 + 23 and 15 + 16 + 23 extra bits: LL code 35,
    # ML code 52 (both fields at their widest cannot fit one 128 KiB block)
    big = rand(140_000, 2)
    prefix = [rle(k & 0xFF, 128 << 10) for k in range(127)]                      # 127 blocks of 128 KiB, values 0..126
    n = 127 << 17
    add("of_code24", frame(prefix + [raw(big[:(1 << 24) - 3 - n - 1]),
                                     comp(lit_raw(big[:1]) + seq_section([(1, 1 << 24, 3)], of=("R", 24)))],
                     1 << 24, single=True))
    half = [rle((k * 7) & 0xFF, 128 << 10) for k in range(66)]                   # 8.25 MiB: offsets of 23 bits
    add("wide_ll", frame(half + [comp(lit_raw(big[:65_540]) + seq_section(
        [(65_536 + 4, (66 << 17) - 9 + 3, 32_771 + 32_000)]))], None, wd=0x78))
    add("wide_ml", frame(half + [comp(lit_raw(big[:32_800]) + seq_section(
        [(32_768 + 32, (66 << 17) - 5 + 3, 65_539 + 30_000)]))], None, wd=0x78))
    # accuracy logs 5..9 (LL, ML) and 5..8 (OF), tables fitted to the block's codes
    s = [(k % 7, 4 + k % 5 + 3 * (k % 3) + 3, 3 + k % 2) for k in range(60)]
    lits = rand(sum(a for a, _, _ in s), 3)
    pre = rand(40, 4)

    def codes(col):
        cs = [seq_codes(a, c, b - 3) for a, b, c in s]
        return sorted({x[(0, 2, 1)[col]][0] for x in cs})
    for log in (5, 6, 7, 8, 9):
        lo = min(log, 8)
        add(f"logs{log}", frame([raw(pre), comp(lit_raw(lits) + seq_section(
            s, ("F", norm_of(codes(0), 36, log), log), ("F", norm_of(codes(1), 32, lo), lo),
            ("F", norm_of(codes(2), 53, log), log)))], None, wd=0x00))
    # RLE_Mode with the largest LL and ML codes (one sequence cannot hold both); OF's is in of_code24
    add("rle_max", frame([raw(rand(200_000, 5)[:128 << 10]), raw(rand(60_000, 6)),
                          comp(lit_raw(big[:65_540]) + seq_section([(65_540, 100_000 + 3, 30)],
                                                                   ("R", 35), ("R", 16), ("R", 27))),
                          comp(lit_raw(big[:10]) + seq_section([(10, 150_000 + 3, 65_539 + 10)],
                                                               ("R", 10), ("R", 17), ("R", 52)))], None, wd=0x78))
    # FSE descriptions with "less than 1" counts, zero runs of 4 and 6 (repeat flags 3, 0 and 3, 2), the largest symbol
    ll_norm = [20, 0, 0, 0, 0, 12, 10, 0, 0, 0, 0, 0, 0, 10] + [0] * 21 + [-1]
    ll_norm[0] += 64 - sum(abs(x) for x in ll_norm)
    of_norm = [0] * 32
    of_norm[2], of_norm[3], of_norm[4], of_norm[31] = 12, 10, 9, -1
    ml_norm = [0] * 53
    ml_norm[0], ml_norm[1], ml_norm[5], ml_norm[52] = 30, 20, 13, -1
    sq = [((0, 5, 6, 13)[k % 4], (5, 9, 17, 3)[k % 4] + 3, (3, 4, 8, 3)[k % 4]) for k in range(16)]
    add("fse_edges", frame([raw(pre), comp(lit_raw(rand(sum(a for a, _, _ in sq), 7)) + seq_section(
        sq, ("F", ll_norm, 6), ("F", of_norm, 5), ("F", ml_norm, 6)))], None, wd=0x00))
    # Repeat_Mode after Predefined, after RLE and after FSE_Compressed, per column
    fl, fm = ("F", norm_of([3, 5], 36, 5), 5), ("F", norm_of([1, 2, 3], 53, 5), 5)
    add("repeat_modes", frame([raw(pre), comp(lit_raw(rand(30, 8)) + seq_section(
        [(5, 10, 4), (3, 12, 5)], ("P",), ("R", 3), fm)),
        comp(lit_raw(rand(16, 9)) + seq_section([(5, 10, 4), (3, 8, 5), (3, 14, 6)], ("X", ("P",)), ("X", ("R", 3)),
                                                ("X", fm))),
        comp(lit_raw(rand(13, 10)) + seq_section([(3, 11, 6), (5, 9, 6)], fl, ("P",), ("R", 3))),
        comp(lit_raw(rand(8, 11)) + seq_section([(3, 9, 6), (5, 10, 6)], ("X", fl), ("X", ("P",)),
                                                ("X", ("R", 3))))], None, wd=0x00))
    # literals: the largest size of each header form
    add("content_128k", frame([comp(lit_raw(big[:(128 << 10) - 4]) + b"\0")], None, wd=0x78))
    add("lit_raw_max", frame([comp(lit_raw(t[:31]) + b"\0"), comp(lit_raw(t[:4095]) + b"\0"),
                              comp(lit_raw(big[:(128 << 10) - 5]) + b"\0"), comp(lit_rle(0x41, 128 << 10) + b"\0")],
                             None, wd=0x78))
    skew = lengths_of({0x61: 1, 0x62: 2, 0x63: 3, 0x64: 3})
    sk = np.random.default_rng(12).choice(np.array([0x61, 0x62, 0x63, 0x64], np.uint8), 128 << 10,
                                          p=[0.5, 0.25, 0.125, 0.125]).tobytes()
    add("lit_huf_max", frame([comp(lit_huf(sk[:1023], skew, streams=1) + b"\0"),
                              comp(lit_huf(sk[:1023], skew, streams=4, sf=1) + b"\0"),
                              comp(lit_huf(sk[:16_383], skew, streams=4, sf=2) + b"\0"),
                              comp(lit_huf(sk, skew, streams=4, sf=3) + b"\0")], None, wd=0x78))
    # four streams of 6..9 literals: the last one holds 0, 0, 0, 1 symbols
    for n4 in (6, 7, 8, 9):
        add(f"huf4x_{n4}", frame([comp(lit_huf(sk[:n4], skew, streams=4) + b"\0")], None, wd=0x00))
    # Treeless literals with 1 and 4 streams, after a block that stated the tree
    add("treeless", frame([comp(lit_huf(sk[:500], skew, "fse") + b"\0"), comp(lit_huf(sk[500:700], skew, None) + b"\0"),
                           comp(lit_huf(sk[700:1900], skew, None, streams=4) + b"\0")], None, wd=0x38))
    # an 11-bit tree: lengths 1..10, 11, 11
    l11 = lengths_of({**{48 + k: k + 1 for k in range(10)}, 58: 11, 59: 11})
    d11 = bytes([48 + k for k in range(10) for _ in range(1 << (9 - k))] + [58, 59, 59, 58]) * 4
    add("huf_11bit", frame([comp(lit_huf(d11, l11, streams=4) + b"\0")], None, wd=0x38))
    # 256 symbols through FSE-compressed weights (255 stated), and 129 through 128 direct weights
    l256 = [8] * 256
    l256[7], l256[200], l256[255] = 7, 9, 9
    d256 = bytes(range(256)) * 6 + bytes([7]) * 9
    add("huf_256sym", frame([comp(lit_huf(d256, l256, "fse", streams=4) + b"\0")], None, wd=0x38))
    l129 = [7] * 127 + [8, 8] + [0] * 127
    add("huf_direct128", frame([comp(lit_huf(bytes(range(129)) * 5, l129, "direct", streams=4) + b"\0")],
                               None, wd=0x00))
    # frame header: every Window_Descriptor mantissa (no Frame_Content_Size, so libzstd checks the window)
    for m in range(1, 8):                                                        # m0: most windowed cases
        add(f"window_m{m}", frame([raw(t[:100]), rle(0x20 + m, 900)], None, wd=m))
    # blocks of exactly Block_Maximum_Size under a 1 KiB window
    add("bmax_1k", frame([raw(t[:1024]), rle(0x55, 1024),
                          comp(lit_raw(t[1024:1521]) + seq_section([(400, 700 + 3, 524), (97, 1, 3)]))],
                         None, wd=0x00))
    # 2-byte Frame_Content_Size at 256 and at 65 791
    add("fcs2_256", frame([raw(t[:256])], 256, single=True))
    add("fcs2_65791", frame([raw(big[:65_536]), rle(0x77, 255)], 65_791, single=True))
    # an empty frame, and a content checksum on a second frame that starts 5 bytes in
    add("empty", frame([raw(b"")], 0, single=True))
    c2 = t[500:600]
    add("checksum_unaligned", frame([raw(t[:5])], 5, single=True) + frame([raw(c2)], None, wd=0x00, checksum=c2))
    return out


def _invalid():
    """(name, payload, chunk_len, status) of every invalid case."""
    out = []
    BAD = _lib.DEC_BAD_FRAME
    add = lambda name, payload, size, st=BAD: out.append((name, payload, size, st))   # noqa: E731
    t = rand(4096, 21)
    hello = [raw(b"hello")]
    # the Window_Size limit of libzstd's streaming decoder (2^27 + 1 bytes)
    add("window_2^28", frame(hello, None, wd=0x90), 5)
    add("window_2^27+2^24", frame(hello, None, wd=0x89), 5)
    add("single_2^27+2", frame([rle(0x11, 1 << 17)], (1 << 27) + 2, single=True), (1 << 27) + 2)
    # header rules
    add("fhd_reserved", frame(hello, None, wd=0x00, fhd_or=8), 5)
    add("dictionary_id", frame(hello, None, wd=0x00, did=b"\x07"), 5)
    add("block_type3", frame([(3, 5, b"hello")], None, wd=0x00), 5)
    add("raw_over_bmax", frame([raw(t[:1025])], None, wd=0x00), 1025)
    add("rle_over_bmax", frame([rle(1, 1025)], None, wd=0x00), 1025)
    body = lit_raw(rand(140_000, 22)[:(128 << 10) - 3]) + b"\0"
    add("content_over_bmax", frame([comp(body)], None, wd=0x78), len(body) - 4)
    add("fcs_differs", frame([raw(b"hello")], 6, single=True), 6)
    add("bad_checksum", frame([raw(t[:50])], None, wd=0x00, checksum=t[1:51]), 50, _lib.DEC_BAD_CHECKSUM)
    add("trailing_bytes", frame(hello, None, wd=0x00) + b"\0\0\0\0", 5)
    add("skippable_truncated", frame(hello, None, wd=0x00) + skippable(20)[:-1], 5)
    add("skippable_header_cut", frame(hello, None, wd=0x00) + skippable(20)[:6], 5)
    # sequences
    s = [(10, 7 + 3, 5), (0, 3, 5)]                                                   # the 2nd: rep0 - 1 = 6
    add("rep0_minus1_zero", frame([comp(lit_raw(t[:11]) + seq_section([(10, 1 + 3, 5), (0, 3, 5), (1, 3, 3)]))],
                                  None, wd=0x00), 24)
    add("offset_beyond", frame([raw(t[:10]), comp(lit_raw(t[:5]) + seq_section([(5, 16 + 3, 4)]))], None, wd=0x00), 19)
    add("literals_overrun", frame([comp(lit_raw(t[:10]) + seq_section([(6, 5 + 3, 4), (6, 5 + 3, 4)]))], None, wd=0x00),
        20)
    add("decoded_over_bmax", frame([comp(lit_raw(t[:100]) + seq_section([(100, 50 + 3, 1000)]))], None, wd=0x00), 1100)
    add("repeat_no_table", frame([comp(lit_raw(t[:10]) + seq_section(s, ("X", ("P",))))], None, wd=0x00), 20)
    add("modes_reserved", frame([comp(lit_raw(t[:10]) + seq_section(s, modes_or=1))], None, wd=0x00), 20)
    sec = bytearray(seq_section(s, ("R", 35)))
    sec[2] = 36
    add("rle_symbol_over", frame([comp(lit_raw(t[:10]) + bytes(sec))], None, wd=0x00), 20)
    add("table_log_over", frame([comp(lit_raw(t[:10]) + seq_section(s, ("F", norm_of([0, 10], 36, 10), 10)))],
                                None, wd=0x00), 20)
    w = _Bits()                          # OF: a zero count, then repeat flags past code 31
    w.add(0, 4); w.add(1, 5)
    for _ in range(11):
        w.add(3, 2)
    add("table_zeros_past_max", frame([comp(lit_raw(t[:10]) + bytes([2, 2 << 4]) + w.flush() + b"\x01")], None,
                                      wd=0x00), 20)
    add("seq_bit_left", frame([comp(lit_raw(t[:10]) + seq_section(s, tweak=lambda b: shift(b, 1)))], None, wd=0x00), 20)
    add("seq_bit_missing", frame([comp(lit_raw(t[:10]) + seq_section(s, tweak=lambda b: shift(b, -1)))], None,
                                 wd=0x00), 20)
    add("seq_no_end_mark", frame([comp(lit_raw(t[:10]) + seq_section(s, tweak=lambda b: b + b"\0"))], None, wd=0x00), 20)
    add("seq_trailing", frame([comp(lit_raw(t[:10]) + b"\0\0")], None, wd=0x00), 10)
    # literals
    skew = lengths_of({0x61: 1, 0x62: 2, 0x63: 3, 0x64: 3})
    d = bytes([0x61, 0x62, 0x61, 0x63, 0x64, 0x61, 0x61, 0x62] * 40)
    add("treeless_no_tree", frame([comp(lit_huf(d, skew, None) + b"\0")], None, wd=0x00), len(d))
    add("huf4x_5", frame([comp(lit_huf(d[:5], skew, streams=4) + b"\0")], None, wd=0x00), 5)
    for k in range(4):
        for by, nm in ((1, "left"), (-1, "missing")):
            tw = (lambda k_, by_: lambda j, p: shift(p, by_) if j == k_ else p)(k, by)
            add(f"huf4x_s{k}_bit_{nm}", frame([comp(lit_huf(d, skew, streams=4, tweak=tw) + b"\0")], None, wd=0x00),
                len(d))
    for by, nm in ((1, "left"), (-1, "missing")):
        add(f"huf1x_bit_{nm}", frame([comp(lit_huf(d, skew, tweak=lambda j, p: shift(p, by)) + b"\0")], None, wd=0x00),
            len(d))
    add("huf_no_end_mark", frame([comp(lit_huf(d, skew, tweak=lambda j, p: p + b"\0") + b"\0")], None, wd=0x00), len(d))
    add("huf_incomplete", frame([comp(lit_huf(d[:20], skew)[:4] + bytes([127 + 3, 0x11, 0x10]) +
                                      lit_huf(d[:20], skew)[6:] + b"\0")], None, wd=0x00), 20)
    l12 = lengths_of({**{48 + k: k + 1 for k in range(11)}, 59: 12, 60: 12})
    d12 = bytes([48 + k for k in range(11) for _ in range(1 << (10 - k))] + [59, 60])
    add("huf_12bit", frame([comp(lit_huf(d12, l12, streams=4) + b"\0")], None, wd=0x38), len(d12))
    add("lit_rle_over_bmax", frame([comp(lit_rle(0x41, 1025) + b"\0")], None, wd=0x00), 1025)
    return out


# Cases whose verdict differs between libzstd 1.5.5's streaming decoder and RFC 8878 as K13 reads it: libzstd reads
# them, K13 and zstd_forms.decode_payload refuse them.  name -> (the size libzstd decodes, why)
_BITS = ("libzstd 1.5.5 does not check that this bitstream is consumed exactly; K13 requires every bit of a stream to "
         "be read, no more and no fewer")
KNOWN_DIFFERENCES = {
    "rep0_minus1_zero": (24, "libzstd 1.5.5 turns the offset 0 that rep0 - 1 gives into 1 in its streaming path (its "
                             "one-shot path refuses it); an offset of 0 is invalid"),
    "modes_reserved": (20, "libzstd 1.5.5 ignores the reserved bits of Symbol_Compression_Modes, which RFC 8878 says "
                           "must be zero"),
    "seq_bit_left": (20, _BITS), "seq_bit_missing": (20, _BITS),
    **{f"huf4x_s{k}_bit_{e}": (320, _BITS) for k in range(4) for e in ("left", "missing")},
    "huf_12bit": (2049, "libzstd accepts Huffman codes of up to 12 bits; RFC 8878 limits them to 11, and K13's "
                        "decoding table has 2^11 entries"),
}


@lru_cache(maxsize=1)
def edge_cases() -> tuple[Case, ...]:
    """Every case, the valid ones first."""
    out = []
    for name, payload in _valid():
        content = zf.decode_payload(payload)
        out.append(Case(name, payload, content, _lib.DEC_OK, len(content)))
    for name, payload, size, st in _invalid():
        out.append(Case(name, payload, None, st, size))
    return tuple(out)
