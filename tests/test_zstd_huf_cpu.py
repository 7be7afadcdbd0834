"""The compressed DataBlob format with full-alphabet Huffman literals (tests/zstd_huf_ref.py: zstd_frame_lzh /
blob_encode_lzh), checked on the CPU against libzstd's decoder (pyarrow's codec): every frame decodes back to its input,
no block is larger than in the _lze frame, and each tree form, weight count and stream layout decodes to what it says."""
import zlib

import numpy as np
import pytest

from oracle import pyref
import zstd_ent_ref as entref
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from test_zstd_ent_cpu import seqs_over
from test_zstd_lz_cpu import PREFIX, blocks, decode, lz_decode, rnd

pa = pytest.importorskip("pyarrow")
B = pyref.ZFRAME_BLOCK


def check(data: bytes):
    """Decodes to the input, no block larger than in zstd_frame_lze (constant blocks stay RLE), deterministic."""
    fr = hufref.zstd_frame_lzh(data)
    assert decode(fr, len(data)) == data
    ref = blocks(entref.zstd_frame_lze(data))
    got = blocks(fr)
    assert len(got) == len(ref)
    for (t, _, n), (t0, _, n0) in zip(got, ref):
        assert n <= n0
        assert (t == 1) == (t0 == 1)
    assert hufref.zstd_frame_lzh(data) == fr
    return fr, got


def huf_frame(lits: bytes, seqs):
    """A frame of a 64-byte Raw_Block and the full-alphabet Block_Content of (lits, seqs) -> (frame, expected output,
    Block_Content)."""
    body = hufref.entropy_block_lzh(lits, seqs)
    want = PREFIX + lz_decode(lits, seqs)
    assert len(body) <= B and len(want) - len(PREFIX) <= B
    hdr = (len(PREFIX) << 3).to_bytes(3, "little") + PREFIX + (1 | 2 << 1 | len(body) << 3).to_bytes(3, "little")
    return b"\x28\xb5\x2f\xfd\xe0" + len(want).to_bytes(8, "little") + hdr + body, want, body


def tree_form(body: bytes):
    """Of a Block_Content with Huffman literals: ("fse" or "direct", the tree description's header byte)."""
    assert body[0] & 3 == 2
    sf = (body[0] >> 2) & 3
    h = body[3 if sf < 2 else sf + 2]
    return ("fse" if h < 128 else "direct"), h


def weights_of(lits: bytes):
    lengths = entref.huf_lengths(np.bincount(np.frombuffer(lits, np.uint8), minlength=256).tolist())
    mx, top = max(lengths), max(s for s in range(256) if lengths[s])
    return [mx + 1 - lengths[s] if lengths[s] else 0 for s in range(top)]


def round_trip(lits: bytes, nseq: int = 20):
    frame, want, body = huf_frame(lits, seqs_over(lits, nseq))
    assert decode(frame, len(want)) == want
    return body


@pytest.mark.parametrize("top", [129, 200, 255])
def test_literals_above_128_are_huffman_coded(top):
    lits = bytearray(bytes(lzref.text_corpus(5000, 2)))
    lits[100] = top
    lits = bytes(lits)
    body = round_trip(lits, 100)
    assert tree_form(body)[0] == "fse"
    assert entref.literals_section(lits)[0] & 3 == 0           # _lze keeps them raw
    assert len(body) < len(entref.entropy_block(lits, seqs_over(lits, 100)))


@pytest.mark.parametrize("top", [2, 3, 4, 5, 130, 131, 254, 255])
def test_odd_and_even_weight_counts(top):
    """top weights are listed; the two states end on different weights for odd and even counts."""
    rng = np.random.default_rng(top)
    p = 1.0 / np.arange(1, top + 2)
    vals = np.concatenate([np.arange(top + 1), rng.choice(top + 1, 4000, p=p / p.sum())]).astype(np.uint8)
    lits = rng.permutation(vals).tobytes()
    assert len(weights_of(lits)) == top
    body = round_trip(lits)
    assert tree_form(body)[0] == "fse" or top <= 128


@pytest.mark.parametrize("vals", [(5, 200), (0, 255), (250, 251, 252, 253)])
def test_exactly_two_distinct_weights(vals):
    """Mostly absent symbols: weight 0 holds more than half of the states, so a state that starts where no bits are
    written would not end the stream (zstd_huf_ref.fse_weights)."""
    lits = np.random.default_rng(len(vals)).choice(np.array(vals, np.uint8), 3000).tobytes()
    assert len(set(weights_of(lits))) == 2
    body = round_trip(lits)
    assert tree_form(body)[0] == "fse"


def test_fse_form_below_129_only_where_it_is_smaller():
    """top <= 128: the FSE form where it beats the direct one (a sparse alphabet, or text), else the frame is _lze's
    (a small dense alphabet)."""
    lits = np.random.default_rng(3).choice(np.array([1, 60, 120], np.uint8), 3000).tobytes()
    body = round_trip(lits)
    form, h = tree_form(body)
    assert form == "fse" and 1 + h < 1 + (120 + 1) // 2
    assert len(body) < len(entref.entropy_block(lits, seqs_over(lits, 20)))
    text = bytes(lzref.text_corpus(B, 4))
    lits, seqs = lzref.lz_parse(text)
    assert max(text) <= 128 and tree_form(hufref.entropy_block_lzh(lits, seqs))[0] == "fse"
    assert len(hufref.zstd_frame_lzh(text)) < len(entref.zstd_frame_lze(text))
    p = np.array([20, 14, 12, 10, 9, 8, 7, 6, 5, 4, 3, 2], float)
    dense = np.random.default_rng(5).choice(12, 3 * B, p=p / p.sum()).astype(np.uint8).tobytes()
    fr, _ = check(dense)
    assert fr == entref.zstd_frame_lze(dense)
    for k in range(3):
        lits, seqs = lzref.lz_parse(dense[k * B:(k + 1) * B])
        assert tree_form(hufref.entropy_block_lzh(lits, seqs))[0] == "direct"


def test_uniform_histogram_has_no_tree_form_and_stays_raw():
    """Every value equally often: one weight for all symbols, which the FSE form cannot state, and top = 255."""
    lits = bytes(range(256)) * 12
    assert set(weights_of(lits)) == {1}
    assert hufref.tree_description(entref.huf_lengths([12] * 256)) is None
    body = hufref.literals_section_lzh(lits)
    assert body[0] & 3 == 0 and body[2:] == lits
    frame, want, _ = huf_frame(lits, [])
    assert decode(frame, len(want)) == want


def test_fse_form_stays_within_its_127_byte_header():
    """The FSE form's header byte states at most 127 bytes; the form is not used beyond that.  With at most 255 weights
    of 12 values, even evenly spread ones (no complete code has them: its many long codes make low weights dominate)
    stay within it, about 3.6 bits a weight."""
    for seed in range(20):
        lengths = np.random.default_rng(seed).integers(0, 12, 256).tolist()
        lengths[255] = 5
        wts = [max(lengths) + 1 - ln if ln else 0 for ln in lengths[:255]]
        fse = hufref.fse_weights(wts)
        assert 100 < len(fse) <= hufref.FSE_TREE_MAX
        assert hufref.tree_description(lengths) == bytes([len(fse)]) + fse


@pytest.mark.parametrize("n_lit", [2, 3, 31, 32, 1023, 1024, 4095, 4096, 16383, 16384, B - 8])
def test_literal_counts_at_stream_and_size_format_edges(n_lit):
    """One stream up to 1023 literals (Size_Format 00), then four streams with 14-bit (10) or 18-bit (11) sizes.  Four
    streams with 10-bit sizes (01) do not occur: below 1024 literals one stream is taken whenever it fits 10 bits."""
    p = [.4, .2, .15, .1, .1, .05]
    lits = (b"\xf0\x81" + np.random.default_rng(n_lit).choice(np.array([0x80, 0xC3, 0xFF, 0x48, 0x89, 0xE8], np.uint8),
                                                              n_lit, p=p).tobytes())[:n_lit]
    frame, want, body = huf_frame(lits, [])
    assert decode(frame, len(want)) == want
    typ, sf = body[0] & 3, (body[0] >> 2) & 3
    if n_lit <= 3:
        assert typ == 0                                        # a tree that costs more than it saves
        return
    assert typ == 2 and tree_form(body)[0] == "fse"
    c = int.from_bytes(body[:5], "little")
    assert (c >> 4) & (0x3FF if sf < 2 else 0x3FFF if sf == 2 else 0x3FFFF) == n_lit
    assert sf == (0 if n_lit <= 1023 else 2 if n_lit <= 16383 else 3)


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 6, 7, 100, B - 1, B, B + 1, 2 * B + 5, 3 * B - 3])
def test_lengths_and_ragged_tails(n):
    data = bytes(hufref.binary_corpus(n, 3)) if n else b""
    fr, got = check(data)
    if n >= 1000:
        assert got[0][0] == 2


def test_periodic_data_with_overlapping_copies():
    seed = rnd(300, 5)
    for period in range(1, 301):
        data = (seed[:period] * (20000 // period + 1))[:20000 - period % 7]
        check(data)


def test_random_data_stays_raw_and_mixtures_shrink():
    data = rnd(3 * B + 1000, 9)
    fr, got = check(data)
    assert fr == pyref.zstd_frame_rle_raw(data)
    assert hufref.blob_encode_lzh(data) == pyref.blob_encode(data)
    binary = bytes(hufref.binary_corpus(3 * B, 11))
    data = binary[:B + 12345] + bytes(3 * B) + rnd(B, 12) + binary[B:2 * B] + b"\xAA" * 5000 + rnd(777, 13)
    fr, got = check(data)
    blob = hufref.blob_encode_lzh(data)
    assert blob[:8] == pyref.BLOB_MAGIC_COMPRESSED and blob[12:] == fr
    assert int.from_bytes(blob[8:12], "little") == zlib.crc32(fr)
    assert len(blob) < len(entref.blob_encode_lze(data))


def test_binary_corpus_takes_the_new_path_and_compresses_below_lze():
    """On most blocks of the binary corpus _lze keeps the literals raw and _lzh Huffman-codes them; DESIGN.md K10 has
    the sizes."""
    data = bytes(hufref.binary_corpus(2 << 20, 1))
    assert bytes(hufref.binary_corpus(2 << 20, 1)) == data
    fr, _ = check(data)
    new = 0
    for k in range(len(data) // B):
        lits, _ = lzref.lz_parse(data[k * B:(k + 1) * B])
        new += entref.literals_section(bytes(lits))[0] & 3 == 0 and hufref.literals_section_lzh(bytes(lits))[0] & 3 == 2
    assert new >= 0.8 * (len(data) // B)
    assert len(fr) < len(entref.zstd_frame_lze(data))
