"""The compressed DataBlob format with zstd's entropy stage (tests/zstd_ent_ref.py: zstd_frame_lze / blob_encode_lze),
checked on the CPU against libzstd's decoder (pyarrow's codec): every frame decodes back to its input, no block is larger
than in the _lz frame, and each literal form, Huffman rule and table mode decodes to what it says."""
import zlib

import numpy as np
import pytest

from oracle import pyref
import zstd_ent_ref as entref
import zstd_lz_ref as lzref
from test_zstd_lz_cpu import PREFIX, blocks, decode, lz_decode, rnd

pa = pytest.importorskip("pyarrow")
B = pyref.ZFRAME_BLOCK


def check(data: bytes):
    """Decodes to the input, no block larger than in zstd_frame_lz (constant blocks stay RLE), deterministic."""
    fr = entref.zstd_frame_lze(data)
    assert decode(fr, len(data)) == data
    ref = blocks(lzref.zstd_frame_lz(data))
    got = blocks(fr)
    assert len(got) == len(ref)
    for (t, _, n), (t0, _, n0) in zip(got, ref):
        assert n <= n0
        assert (t == 1) == (t0 == 1)
    assert entref.zstd_frame_lze(data) == fr
    return fr, got


def ent_frame(lits: bytes, seqs):
    """A frame of a 64-byte Raw_Block and the entropy-coded Block_Content of (lits, seqs) (see
    test_zstd_lz_cpu.one_block_frame) -> (frame, expected output, Block_Content)."""
    body = entref.entropy_block(lits, seqs)
    want = PREFIX + lz_decode(lits, seqs)
    assert len(body) <= B and len(want) - len(PREFIX) <= B
    hdr = (len(PREFIX) << 3).to_bytes(3, "little") + PREFIX + (1 | 2 << 1 | len(body) << 3).to_bytes(3, "little")
    return b"\x28\xb5\x2f\xfd\xe0" + len(want).to_bytes(8, "little") + hdr + body, want, body


def lit_form(body: bytes):
    """(Literals_Block_Type, Size_Format) of a Block_Content."""
    return body[0] & 3, (body[0] >> 2) & 3


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 6, 7, 100, B - 1, B, B + 1, 2 * B + 5, 3 * B - 3])
def test_lengths_and_ragged_tails(n):
    data = bytes(lzref.text_corpus(n, 3)) if n else b""
    fr, got = check(data)
    if n >= 1000:
        assert got[0][0] == 2


def test_periodic_data_with_overlapping_copies():
    seed = rnd(300, 5)
    for period in range(1, 301):
        data = (seed[:period] * (20000 // period + 1))[:20000 - period % 7]
        check(data)


def test_one_match_spans_a_whole_block():
    data = b"\x01\x02\x03\x04" * (B // 4)
    fr, got = check(data + rnd(B, 6))
    assert got[0][0] == 2
    lits, seqs = lzref.lz_parse(data)
    assert len(seqs) == 1
    frame, want, body = ent_frame(lits, seqs)
    assert decode(frame, len(want)) == want


def test_random_data_stays_raw_and_mixtures_shrink():
    data = rnd(3 * B + 1000, 9)
    fr, got = check(data)
    assert fr == pyref.zstd_frame_rle_raw(data)
    assert entref.blob_encode_lze(data) == pyref.blob_encode(data)
    text = bytes(lzref.text_corpus(3 * B, 11))
    data = text[:B + 12345] + bytes(3 * B) + rnd(B, 12) + text[B:2 * B] + b"\xAA" * 5000 + rnd(777, 13)
    fr, got = check(data)
    blob = entref.blob_encode_lze(data)
    assert blob[:8] == pyref.BLOB_MAGIC_COMPRESSED and blob[12:] == fr
    assert int.from_bytes(blob[8:12], "little") == zlib.crc32(fr)
    assert len(blob) < len(lzref.blob_encode_lz(data))


def seqs_over(lits: bytes, n: int, ml: int = 4, off: int = 2):
    """n sequences that spread the literals evenly and copy ml bytes from `off` back."""
    k = len(lits) // n
    return [(k + (len(lits) - k * n if i == 0 else 0), ml, off) for i in range(n)]


def test_rle_literals():
    lits = b"\x61" * 500
    frame, want, body = ent_frame(lits, seqs_over(lits, 50))
    assert lit_form(body) == (1, 1) and body[2] == 0x61
    assert decode(frame, len(want)) == want
    for n_lit in (1, 31, 32, 4095, 4096):
        frame, want, body = ent_frame(b"\x07" * n_lit, [])
        assert body[0] & 3 == 1 and len(body) == (1 if n_lit <= 31 else 2 if n_lit <= 4095 else 3) + 2
        assert decode(frame, len(want)) == want


def test_two_literal_values():
    lits = np.random.default_rng(1).choice(np.array([3, 200 - 100], np.uint8), 3000).tobytes()
    frame, want, body = ent_frame(lits, seqs_over(lits, 20))
    assert body[0] & 3 == 2
    assert decode(frame, len(want)) == want


@pytest.mark.parametrize("top,kind", [(128, 2), (129, 0)])
def test_largest_literal_value_128_uses_huffman_and_129_stays_raw(top, kind):
    lits = bytearray(bytes(lzref.text_corpus(5000, 2)))
    lits[100] = top
    frame, want, body = ent_frame(bytes(lits), seqs_over(bytes(lits), 100))
    assert body[0] & 3 == kind
    assert decode(frame, len(want)) == want


@pytest.mark.parametrize("n_lit", [1, 2, 31, 32, 1023, 1024, 4095, 4096, 16383, 16384, B - 8])
def test_literal_counts_at_stream_and_size_format_edges(n_lit):
    """One stream up to 1023 literals (Size_Format 00), then four streams with 14-bit (10) or 18-bit (11) sizes."""
    lits = (b"\0\1" + np.random.default_rng(n_lit).choice(np.arange(6, dtype=np.uint8), n_lit,
                                                         p=[.4, .2, .15, .1, .1, .05]).tobytes())[:n_lit]
    frame, want, body = ent_frame(lits, [])
    assert decode(frame, len(want)) == want
    typ, sf = lit_form(body)
    if n_lit <= 2:
        assert typ == (1 if n_lit == 1 else 0)                # one value; a tree that costs more than it saves
        return
    assert typ == 2
    c = int.from_bytes(body[:5], "little")
    size = (c >> 4) & (0x3FF if sf < 2 else 0x3FFF if sf == 2 else 0x3FFFF)
    assert size == n_lit
    assert sf == (0 if n_lit <= 1023 else 2 if n_lit <= 16383 else 3)


def test_huffman_literals_only_when_smaller_than_raw():
    """129 distinct values once each: the tree description alone outweighs the saving, so the literals stay raw."""
    lits = bytes(range(129))
    assert len(entref.huffman_literals(np.frombuffer(lits, np.uint8), np.bincount(np.frombuffer(lits, np.uint8),
                                                                                     minlength=256).tolist())) > 131
    body = entref.literals_section(lits)
    assert body[0] & 3 == 0 and body[2:] == lits
    lits = np.repeat(np.arange(100, dtype=np.uint8), 10).tobytes()
    body = entref.literals_section(lits)
    assert lit_form(body) == (2, 0)


def test_huffman_lengths_are_limited_to_11_bits():
    fib = [1, 1]
    while len(fib) < 20:
        fib.append(fib[-1] + fib[-2])
    counts = fib + [0] * (256 - len(fib))
    assert max(entref._huffman(counts)) > entref.HUF_MAXBITS
    lengths = entref.huf_lengths(counts)
    assert max(lengths) <= entref.HUF_MAXBITS
    assert sum(2.0 ** -ln for ln in lengths if ln) == 1.0      # complete
    lits = np.random.default_rng(5).permutation(np.repeat(np.arange(20, dtype=np.uint8), fib)).tobytes()
    frame, want, body = ent_frame(lits, seqs_over(lits, 7))
    assert body[0] & 3 == 2
    assert decode(frame, len(want)) == want


def test_normalisation_decrement_and_increment_paths():
    down = [1000] + [1] * 31                                  # 31 cells of 1 on top of 1000 * 512 / 1031
    norm = entref.normalize(down, 9)
    assert sum(max(1, c * 512 // 1031) for c in down) > 512 and sum(norm) == 512 and min(norm) == 1
    up = [3, 3, 3]
    norm = entref.normalize(up, 5)
    assert sum(c * 32 // 9 for c in up) < 32 and norm == [12, 10, 10]
    lits = rnd(40, 30)
    seqs = [(40, 3, 1)] + [(0, 3, 1)] * 999 + [(0, 4 + k, 2) for k in range(31)]   # ML codes 0 x 1000, 1..31 once
    frame, want, body = ent_frame(lits, seqs)
    assert decode(frame, len(want)) == want
    seqs = [(40, 3, 1)] + [(0, 3 + k % 3, 1) for k in range(8)]
    frame, want, body = ent_frame(lits, seqs)
    assert decode(frame, len(want)) == want


def test_rle_mode_when_every_sequence_has_one_code():
    lits = rnd(1, 31) + b"\x01" * 600
    seqs = [(1, 4, 1)] * 600
    frame, want, body = ent_frame(lits, seqs)
    sec = entref.sequences_section(seqs)
    assert sec[2] == 0b01010100                               # LL, OF, ML all RLE_Mode
    assert decode(frame, len(want)) == want


def test_single_sequence():
    lits = rnd(20, 32)
    for seqs in ([(5, 10, 3)], [(20, 65539, 1)], [(0, 3, 1)]):
        frame, want, body = ent_frame(lits if seqs[0][0] else rnd(1, 33), seqs if seqs[0][0] else [(1, 3, 1)])
        assert decode(frame, len(want)) == want


def test_every_code_of_each_table_round_trips():
    lls = [lzref.LL_BASE[c] for c in range(36)]
    mls = [lzref.ML_BASE[c] for c in range(53)]
    seqs, used = [], 4
    for ll, ml in zip(lls + [0] * 17, mls):
        if used + ll + ml > B - 64:
            ll, ml = 0, 3
        off = min(used + ll, 1 << (len(seqs) % 16))
        seqs.append((ll, ml, max(off, 1)))
        used += ll + ml
    lits = bytes(lzref.text_corpus(sum(s[0] for s in seqs) + 4, 23))
    seqs[0] = (seqs[0][0] + 4, seqs[0][1], 1)
    frame, want, body = ent_frame(lits, seqs)
    assert decode(frame, len(want)) == want


def test_text_corpus_compresses_below_the_floor():
    """The committed text + records corpus: 0.346 of the input (DESIGN.md K10), against 0.498 for _lz."""
    data = bytes(lzref.text_corpus(2 << 20, 1))
    fr, _ = check(data)
    assert len(fr) / len(data) <= 0.40
