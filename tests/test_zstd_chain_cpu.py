"""The _lzc restatement (tests/zstd_chain_ref.py) on the CPU: every frame decodes to its input through libzstd's
streaming decoder; offsets reach exactly CH_MAXDIST and no further; matches overlap their source and reach into earlier
blocks; and the chosen constants are pinned by frame size / input against libzstd level 3 and against _lzh."""
import ctypes

import numpy as np
import pytest

import zstd_chain_ref as ch
import zstd_forms as zf
import zstd_huf_ref as hufref
import zstd_ldm_ref as ldm
import zstd_lz_ref as lzref
import zstd_stream_ref as zs
from oracle import pyref
from test_zstd_ldm_cpu import far_copy

B = pyref.ZFRAME_BLOCK


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def earlier_block_copies(seed: int = 10) -> np.ndarray:
    """A random block, then a block of 60-byte pieces of it, each followed by one 0xAA byte: every match's source lies
    in the block before, and the literals between them are all one value (RLE literals)."""
    r = rnd(B, seed)
    pieces = [np.concatenate([r[k * 97:k * 97 + 60], [0xAA]]) for k in range(B // 61)]
    return np.concatenate([r] + pieces).astype(np.uint8)


def overlapping() -> np.ndarray:
    """Periods of 1-7 bytes repeated far beyond their length, between random bytes: every match overlaps its source."""
    rng = np.random.default_rng(11)
    parts = []
    for p in (1, 2, 3, 5, 7):
        parts += [rnd(300, p), np.tile(rng.integers(0, 256, p, dtype=np.uint8), 4000 // p)]
    return np.concatenate(parts)


def small_parts() -> list[np.ndarray]:
    """Chunks of 0-5 bytes, sizes off the block grid, all-constant and half-constant chunks, and the copy cases."""
    text = lzref.text_corpus(3 * B + 777, 12)
    return [text[:k] for k in range(6)] + [
        text[:B - 1], text[:B + 1], text, np.zeros(2 * B + 5, np.uint8), np.full(B, 0xAA, np.uint8),
        np.concatenate([text[:B // 2], np.zeros(B + B // 2, np.uint8), text[B:B + 1000]]),
        earlier_block_copies(), overlapping(), ldm.repeated_image(hufref.binary_corpus(B, 13), 3, 50, 14),
        ch.half_zero(3 * B, 15)]


def census_parts() -> list[np.ndarray]:
    """small_parts() and tests/zstd_forms.py's form parts: together they reach every form REQUIRED_LZC names."""
    return small_parts() + zf.form_parts()


# The forms _lzc frames reach: raw, RLE and compressed blocks; raw, RLE and Huffman literals with 1 and 4 streams;
# sequence tables in RLE and FSE_Compressed mode.
REQUIRED_LZC = {"block:raw", "block:rle", "block:compressed", "lit:raw/1B", "lit:raw/2B", "lit:raw/3B", "lit:rle/2B",
                "lit:huf/sf0", "lit:huf/sf2", "lit:huf/sf3", "modes:FFF", "modes:FRF", "modes:RFF", "nseq:1B", "nseq:2B"}


@pytest.fixture(scope="module")
def stream():
    zs.require()


def test_small_parts_decode_and_are_no_larger_than_lzh(stream):
    for k, p in enumerate(small_parts()):
        d = p.tobytes()
        fr = ch.zstd_frame_lzc(d)
        assert zs.stream_decode(fr) == d, k
        assert len(fr) <= len(hufref.zstd_frame_lzh(d)), k
        blob = ch.blob_encode_lzc(d)
        assert blob[12:] == (fr if d and len(fr) < len(d) else d), k


def test_offsets_reach_maxdist_and_no_further(stream):
    """A 16 MiB chunk with a 1 KiB copy exactly CH_MAXDIST back is one match; one byte further it stays literals."""
    at, beyond = far_copy(ch.CH_MAXDIST), far_copy(ch.CH_MAXDIST + 1)
    assert len(at) > 16 << 20
    f_at, f_beyond = ch.zstd_frame_lzc(at.tobytes()), ch.zstd_frame_lzc(beyond.tobytes())
    assert zs.stream_decode(f_at) == at.tobytes() and zs.stream_decode(f_beyond) == beyond.tobytes()
    assert len(f_at) < len(f_beyond) - 900
    s = ch._Search(at.tobytes(), ch.CH_DEPTH, ch.CH_MINMATCH, ch.CH_MAXDIST)
    blk = ch.CH_MAXDIST // B * B   # the copy starts 4 bytes before the end of this block
    seqs = ch.chain_parse(s, blk, blk + B)[1] + ch.chain_parse(s, blk + B, min(len(at), blk + 2 * B))[1]
    assert sum(L for _, L, o in seqs if o == ch.CH_MAXDIST) >= 1000


def test_matches_overlap_and_reach_earlier_blocks(stream):
    for data, want in ((overlapping(), "overlap"), (earlier_block_copies(), "earlier")):
        d = data.tobytes()
        s = ch._Search(d, ch.CH_DEPTH, ch.CH_MINMATCH, ch.CH_MAXDIST)
        seen = set()
        for b in range(0, len(d), B):
            _, seqs = ch.chain_parse(s, b, min(len(d), b + B))
            pos = b
            for ll, L, o in seqs:
                pos += ll
                if o < L:
                    seen.add("overlap")
                if pos - o < b:
                    seen.add("earlier")
                pos += L
        assert want in seen
        assert zs.stream_decode(ch.zstd_frame_lzc(d)) == d


def test_census_of_the_lzc_forms():
    frames = [ch.zstd_frame_lzc(p.tobytes()) for p in census_parts()]
    c = zf.census(frames)
    assert not REQUIRED_LZC - set(c), sorted(REQUIRED_LZC - set(c))


def _zstd_level(data: bytes, level: int) -> int:
    L = ctypes.CDLL("libzstd.so.1")
    L.ZSTD_compressBound.restype = ctypes.c_size_t
    L.ZSTD_compressBound.argtypes = [ctypes.c_size_t]
    L.ZSTD_compress.restype = ctypes.c_size_t
    L.ZSTD_compress.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    out = ctypes.create_string_buffer(L.ZSTD_compressBound(len(data)))
    n = L.ZSTD_compress(out, len(out), data, len(data), level)
    assert n < len(out)
    return n


@pytest.mark.parametrize("n", [1 << 20, 2 << 20])
@pytest.mark.parametrize("corpus", ["text", "binary"])
def test_constants_beat_libzstd_level_3(stream, corpus, n):
    """CH_DEPTH, CH_LAZY, CH_MARGIN and CH_MINMATCH as chosen in DESIGN.md K16: smaller than libzstd level 3 and than
    _lzh on both corpora, seed 1."""
    d = (lzref.text_corpus(n, 1) if corpus == "text" else hufref.binary_corpus(n, 1)).tobytes()
    fr = ch.zstd_frame_lzc(d)
    assert zs.stream_decode(fr) == d
    assert len(fr) < _zstd_level(d, 3)
    assert len(fr) <= len(hufref.zstd_frame_lzh(d))
