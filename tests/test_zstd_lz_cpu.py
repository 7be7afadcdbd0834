"""The compressed DataBlob format with a match stage (tests/zstd_lz_ref.py: zstd_frame_lz / blob_encode_lz), checked on the
CPU against libzstd's decoder (pyarrow's codec): every frame decodes back to its input, every header form and extreme
code of the block writer decodes to what its sequences say, and no block is larger than in the RLE / raw frame."""
import zlib

import numpy as np
import pytest

from oracle import pyref
import zstd_lz_ref as lzref

pa = pytest.importorskip("pyarrow")
B = pyref.ZFRAME_BLOCK


def decode(frame: bytes, size: int) -> bytes:
    return pa.Codec("zstd").decompress(frame, decompressed_size=size).to_pybytes() if size else b""


def blocks(frame: bytes):
    """(Block_Type, Block_Size, bytes in the frame) of every block of a frame with the 13-byte header."""
    out, p = [], 13
    while True:
        h = int.from_bytes(frame[p:p + 3], "little")
        typ, size = (h >> 1) & 3, h >> 3
        n = 1 if typ == 1 else size
        out.append((typ, size, 3 + n))
        p += 3 + n
        if h & 1:
            assert p == len(frame)
            return out


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def check(data: bytes):
    """Decodes to the input, no block larger than in zstd_frame_rle_raw, and the same bytes on a second run."""
    fr = lzref.zstd_frame_lz(data)
    assert decode(fr, len(data)) == data
    ref = blocks(pyref.zstd_frame_rle_raw(data))
    got = blocks(fr)
    assert len(got) == len(ref)
    for (t, _, n), (t0, _, n0) in zip(got, ref):
        assert n <= n0
        assert (t == 1) == (t0 == 1)                      # constant blocks stay RLE, nothing else becomes RLE
    assert lzref.zstd_frame_lz(data) == fr
    return fr, got


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
        fr, got = check(data)
        if period > 1:
            assert got[0][0] == 2 and got[0][2] < 400 + period, period


def test_one_match_spans_a_whole_block():
    data = b"\x01\x02\x03\x04" + b"\x01\x02\x03\x04" * (B // 4 - 1)
    lits, seqs = lzref.lz_parse(data)
    T = lzref.LZ_TILE                                       # the first tile has no earlier tile to match against
    assert lits == data[:T] and seqs == [(T, B - T, 4)]
    fr, got = check(data + rnd(B, 6))
    assert got[0][0] == 2 and got[0][2] < T + 20


def test_largest_in_block_offset():
    head = rnd(8, 7)
    data = head + bytes(B - 16) + head                      # nothing else in the block hashes like the head
    lits, seqs = lzref.lz_parse(data)
    assert seqs[-1][1:] == (8, B - 8)
    _, _, (oc, _, ob) = lzref.seq_codes(*seqs[-1])
    assert oc == ob == 16
    check(data)
    check(data + head)                                      # the match does not cross into the next block


def test_random_data_falls_back_to_raw_blocks():
    data = rnd(3 * B + 1000, 9)
    fr, got = check(data)
    assert [t for t, _, _ in got] == [0, 0, 0, 0]
    assert fr == pyref.zstd_frame_rle_raw(data)
    assert lzref.blob_encode_lz(data) == pyref.blob_encode(data)


def test_zero_runs_stay_rle():
    data = bytes(2 * B) + b"\x07" * B + bytes(1)
    fr, got = check(data)
    assert [t for t, _, _ in got] == [1, 1, 1, 1]
    assert fr == pyref.zstd_frame_rle_raw(data)


def test_mixtures():
    text = bytes(lzref.text_corpus(3 * B, 11))
    data = text[:B + 12345] + bytes(3 * B) + rnd(B, 12) + text[B:2 * B] + b"\xAA" * 5000 + rnd(777, 13)
    fr, got = check(data)
    assert {t for t, _, _ in got} == {1, 2}
    blob = lzref.blob_encode_lz(data)
    assert blob[:8] == pyref.BLOB_MAGIC_COMPRESSED and blob[12:] == fr
    assert int.from_bytes(blob[8:12], "little") == zlib.crc32(fr)
    assert len(blob) < len(pyref.blob_encode(data))


def lz_decode(lits: bytes, seqs) -> bytes:
    out, p = bytearray(), 0
    for ll, ml, off in seqs:
        out += lits[p:p + ll]
        p += ll
        for _ in range(ml):
            out.append(out[-off])
    return bytes(out + lits[p:])


PREFIX = rnd(64, 19)


def one_block_frame(lits: bytes, seqs) -> tuple[bytes, bytes]:
    """A frame of a 64-byte Raw_Block and the Compressed_Block of (lits, seqs): the prefix makes the window (the
    frame's content size) large enough for a block that is larger than what it decodes to."""
    body = lzref.compressed_block(lits, seqs)
    want = PREFIX + lz_decode(lits, seqs)
    assert len(body) <= B and len(want) - len(PREFIX) <= B
    hdr = (len(PREFIX) << 3).to_bytes(3, "little") + PREFIX + (1 | 2 << 1 | len(body) << 3).to_bytes(3, "little")
    return b"\x28\xb5\x2f\xfd\xe0" + len(want).to_bytes(8, "little") + hdr + body, want


@pytest.mark.parametrize("n_seq", [0, 1, 127, 128, 0x7EFF, 0x7F00, 0x7F00 + 1000])
def test_block_writer_sequence_count_forms(n_seq):
    lits = rnd(4, 20)
    seqs = [(4, 3, 1)] + [(0, 3, 1 + k % 4) for k in range(n_seq - 1)] if n_seq else []
    body = lzref.compressed_block(lits, seqs)
    cnt = body[1 + 4:]
    if n_seq < 128:
        assert cnt[0] == n_seq
    elif n_seq < 0x7F00:
        assert ((cnt[0] - 0x80) << 8) + cnt[1] == n_seq
    else:
        assert cnt[0] == 0xFF and cnt[1] + (cnt[2] << 8) + 0x7F00 == n_seq
    fr, want = one_block_frame(lits, seqs)
    assert decode(fr, len(want)) == want


@pytest.mark.parametrize("n_lit", [0, 31, 32, 4095, 4096, B - 4])
def test_block_writer_literal_size_forms(n_lit):
    lits = rnd(n_lit, 21)
    hl = 1 if n_lit <= 31 else 2 if n_lit <= 4095 else 3
    body = lzref.compressed_block(lits, [])
    assert len(body) == hl + n_lit + 1 and body[hl:hl + n_lit] == lits
    fr, want = one_block_frame(lits, [])
    assert decode(fr, len(want)) == want
    if 0 < n_lit < B - 100:
        fr, want = one_block_frame(lits, [(n_lit, 5, 1), (0, 4, n_lit)])
        assert decode(fr, len(want)) == want


@pytest.mark.parametrize("seqs,tail", [
    ([(65536, 3, 1)], 3),                                   # Literals_Length code 35
    ([(100000, 3, 1), (5, 9, 7)], 3),
    ([(1, B - 1, 1)], 0),                                   # Match_Length code 52
    ([(2, 65539, 2), (0, 3, 1)], 3),
    ([(4, B - 7, 1), (0, 3, B - 3)], 0),                    # Offset code 17: Offset_Value 2^17, the block's whole output
    ([(16, 35, 16), (63, 131, 64), (64, 259, 128), (15, 34, 1)], 3),   # first codes with extra bits
])
def test_block_writer_extreme_codes(seqs, tail):
    lits = rnd(sum(ll for ll, _, _ in seqs) + tail, 22)
    fr, want = one_block_frame(lits, seqs)
    assert decode(fr, len(want)) == want


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
    lits = rnd(sum(s[0] for s in seqs) + 4, 23)
    seqs[0] = (seqs[0][0] + 4, seqs[0][1], 1)
    fr, want = one_block_frame(lits, seqs)
    assert decode(fr, len(want)) == want


def test_text_corpus_compresses_below_the_floor():
    """The committed text + records corpus: 0.498 of the input with these constants (DESIGN.md K9)."""
    data = bytes(lzref.text_corpus(1 << 20, 1))
    assert lzref.text_corpus(1 << 20, 1).tobytes() == data
    fr, _ = check(data)
    assert len(fr) / len(data) < 0.51
