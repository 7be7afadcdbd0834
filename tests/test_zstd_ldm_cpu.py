"""The compressed DataBlob format with long-distance matches (tests/zstd_ldm_ref.py: zstd_frame_lzl / blob_encode_lzl),
checked on the CPU against libzstd's decoder (pyarrow's codec): every frame decodes back to its input, no blob is larger
than its _lzh blob, a block without long spans is _lzh's block, and far repeats are found."""
import zlib

import numpy as np
import pytest

from oracle import pyref
import zstd_forms as zf
import zstd_huf_ref as hufref
import zstd_ldm_ref as ldm
import zstd_lz_ref as lzref
from test_zstd_forms_cpu import gpu_inputs
from test_zstd_lz_cpu import decode, rnd

pa = pytest.importorskip("pyarrow")
B = pyref.ZFRAME_BLOCK
LENGTHS = [0, 1, 3, 4, 5, 6, 7, 63, 64, 100, B - 1, B, B + 1, 2 * B + 5, 3 * B - 3]


def block_bytes(frame: bytes) -> list[bytes]:
    """Every block of a frame with the 13-byte header, header included."""
    out, p = [], 13
    while True:
        h = int.from_bytes(frame[p:p + 3], "little")
        typ, size = (h >> 1) & 3, h >> 3
        n = 3 + (1 if typ == 1 else size)
        out.append(frame[p:p + n])
        p += n
        if h & 1:
            return out


def check(data: bytes):
    """Decodes to the input; blob at most _lzh's; blocks without spans equal _lzh's, the others are no larger."""
    data = bytes(data)
    fr = ldm.zstd_frame_lzl(data)
    assert decode(fr, len(data)) == data
    ref = hufref.zstd_frame_lzh(data)
    spans = ldm.block_spans(data)
    got, want = block_bytes(fr), block_bytes(ref)
    assert len(got) == len(want) == len(spans)
    for g, w, s in zip(got, want, spans):
        if not s:
            assert g == w
        assert len(g) <= len(w)
    assert len(ldm.blob_encode_lzl(data)) <= len(hufref.blob_encode_lzh(data))
    return fr, spans


def anchored_period(n: int, period: int = 64) -> np.ndarray:
    """A chunk repeating `period` random bytes, from the first seed whose period has an anchor: one long match from
    byte `period` to the end."""
    for seed in range(1000):
        r = np.random.default_rng(seed).integers(0, 256, period, dtype=np.uint8)
        d = np.tile(r, n // period + 2)[:n]
        if len(ldm.anchors(d[:4 * period])[0]):
            return d
    raise AssertionError("no seed")


def far_copy(dist: int, n: int = 1024, seed: int = 40) -> np.ndarray:
    """Zeros with n random bytes at 0 and again at `dist`."""
    r = np.frombuffer(rnd(n, seed), np.uint8)
    d = np.zeros(dist + n + 3000, np.uint8)
    d[:n] = r
    d[dist:dist + n] = r
    return d


def ldm_parts() -> list[np.ndarray]:
    """Chunks whose long matches cross one and several block edges, run through constant blocks, overlap their source,
    cover whole blocks, and repeat near-copies of a binary image."""
    binary = hufref.binary_corpus(300_000, 41)
    text = lzref.text_corpus(200_000, 42)
    one_edge = np.concatenate([text[:150_000], rnd_arr(B - 150_000 - 500 + 400_000, 43), text[:1000], text[150_000:]])
    several = np.concatenate([binary, binary, binary[:250_000]])
    x = np.concatenate([text[:180_000], np.zeros(3 * B, np.uint8), binary[:70_000]])
    through_const = np.concatenate([x, x[5:]])
    periodic = anchored_period(3 * B + 999, 300)
    edited = np.concatenate([binary, binary])
    edited[300_000 + np.arange(100, 300_000, 4999)] ^= 0x5A
    return [one_edge, several, through_const, periodic, anchored_period(2 * B + 77), edited,
            ldm.repeated_image(hufref.binary_corpus(400_000, 44), 3, 300, 45)]


def rnd_arr(n, seed):
    return np.frombuffer(rnd(n, seed), np.uint8)


def test_gear_table_and_hash():
    assert int(ldm.gear_table(0)[0]) == 0xE220A8397B1DCDAF          # splitmix64(0)'s first output
    a = rnd_arr(300, 1)
    h = ldm.gear_hashes(a)
    G = [int(g) for g in ldm.GEAR]
    for i in (63, 64, 150, 299):
        x = 0
        for b in a[i - 63:i + 1]:
            x = ((x << 1) + G[b]) & ((1 << 64) - 1)
        assert int(h[i]) == x
    for v in range(256):                                           # no run of one byte value has an anchor
        assert (-G[v]) % (1 << 64) >> (64 - ldm.LDM_RATE) != 0


@pytest.mark.parametrize("n", LENGTHS)
def test_lengths_and_ragged_tails(n):
    check(lzref.text_corpus(n, 3).tobytes() if n else b"")
    check(hufref.binary_corpus(n, 3).tobytes() if n else b"")


def test_random_and_constant_data():
    data = rnd(3 * B + 1000, 9)
    fr, spans = check(data)
    assert fr == pyref.zstd_frame_rle_raw(data) and not any(spans)
    data = bytes(2 * B) + b"\x07" * B + bytes(1)
    fr, spans = check(data)
    assert fr == pyref.zstd_frame_rle_raw(data) and not any(spans)


@pytest.mark.parametrize("k", range(7))
def test_long_match_cases(k):
    data = ldm_parts()[k].tobytes()
    fr, spans = check(data)
    assert any(spans)
    assert len(fr) < len(hufref.zstd_frame_lzh(data))


def test_matches_cross_block_edges_and_skip_constant_blocks():
    parts = ldm_parts()
    kept = ldm.select(ldm.long_matches(parts[1]))                 # three copies of 300 000 bytes
    assert any(e // B - s // B >= 2 for s, e, _ in kept)
    x_len = 180_000 + 3 * B + 70_000                               # x, then x without its first 5 bytes
    kept = ldm.select(ldm.long_matches(parts[2]))
    assert any(s < x_len + 180_000 and e > x_len + 180_000 + 3 * B - 5 for s, e, _ in kept)
    data = parts[2].tobytes()
    spans = ldm.block_spans(data)
    for b, s in enumerate(spans):
        blk = data[b * B:(b + 1) * B]
        assert not (s and blk.count(blk[:1]) == len(blk))


def test_one_span_covers_the_chunk_after_its_first_64_bytes():
    data = anchored_period(2 * B + 77).tobytes()
    assert ldm.select(ldm.long_matches(np.frombuffer(data, np.uint8))) == [(64, len(data), 64)]
    fr, spans = check(data)
    assert spans[0] == [(64, B - 64, 64)] and spans[1] == [(0, B, 64)]
    lits, seqs = ldm.lz_parse_spans(data[B:2 * B], spans[1])
    assert lits == b"" and seqs == [(0, B, 64)]
    w = zf.walk(fr)
    assert "lit:raw/1B" in zf.forms(w[1]) and "nseq:1B" in zf.forms(w[1])


@pytest.mark.parametrize("extra", [0, 1])
def test_source_at_the_largest_offset(extra):
    """A copy exactly LDM_MAXDIST back is found (Offset_Value 2^24 - 1); one byte further it is not."""
    data = far_copy(ldm.LDM_MAXDIST + extra)
    kept = ldm.select(ldm.long_matches(data))
    if extra:
        assert kept == []
    else:
        assert kept[0][0] == ldm.LDM_MAXDIST and kept[0][2] == ldm.LDM_MAXDIST
        _, _, (oc, ov, ob) = lzref.seq_codes(0, 64, ldm.LDM_MAXDIST)
        assert oc == 23 and ov + (1 << oc) == (1 << 24) - 1
    fr, spans = check(data.tobytes())
    assert any(spans) != bool(extra)


def test_overlapping_periodic_copies():
    seed = rnd(300, 5)
    for period in (1, 2, 3, 7, 64, 65, 200, 300):
        data = (seed[:period] * ((3 * B) // period + 1))[:3 * B - period % 7]
        check(data)


def test_selection_rule():
    """(s, e descending, offset); s' = max(s, cur); kept when >= LDM_MINMATCH; cur = e."""
    m = [(100, 300, 9), (100, 300, 5), (100, 200, 1), (250, 330, 2), (250, 400, 3), (500, 563, 4), (600, 700, 6)]
    assert ldm.select(m) == [(100, 300, 5), (300, 400, 3), (600, 700, 6)]


def test_span_parse_cuts_short_matches():
    """A match that reaches into a span is cut at the span's start, and dropped when that leaves fewer than
    LZ_MINMATCH bytes (its first byte is then a literal)."""
    blk = bytes(lzref.text_corpus(B, 46))
    _, seqs = lzref.lz_parse(blk)
    pos = 0
    for ll, ml, _ in seqs:                                         # a match of >= 10 bytes after the first tiles
        pos += ll
        if pos > 1000 and ml >= 10:
            break
        pos += ml
    for cut in (3, 4, 5):
        ss = pos + cut
        lits, s2 = ldm.lz_parse_spans(blk, [(ss, 100, 7)])
        starts, p = [], 0
        for ll, ml, off in s2:
            p += ll
            starts.append((p, ml, off))
            p += ml
        assert (ss, 100, 7) in starts
        assert ((pos, cut) in [(q, ml) for q, ml, _ in starts]) == (cut >= lzref.LZ_MINMATCH)
        assert all(ml >= lzref.LZ_MINMATCH for _, ml, _ in s2)
        assert len(lits) + sum(ml for _, ml, _ in s2) == len(blk)


def test_repeated_binary_image_finds_the_far_copies():
    """4 copies of 1 MiB of binary_corpus with 2000 random byte edits: about 0.2 of the input (DESIGN.md K12), where
    _lzh stores 0.75."""
    data = ldm.repeated_image(hufref.binary_corpus(1 << 20, 1)).tobytes()
    fr, _ = check(data)
    assert len(fr) / len(data) <= 0.25


def test_blob_layout():
    data = ldm_parts()[1].tobytes()
    fr = ldm.zstd_frame_lzl(data)
    blob = ldm.blob_encode_lzl(data)
    assert blob[:8] == pyref.BLOB_MAGIC_COMPRESSED and blob[12:] == fr
    assert int.from_bytes(blob[8:12], "little") == zlib.crc32(fr)
    assert ldm.blob_encode_lzl(rnd(5000, 2)) == pyref.blob_encode(rnd(5000, 2))
    assert ldm.blob_encode_lzl(b"") == pyref.blob_encode(b"")


REQUIRED_LZL = zf.REQUIRED["lzh"] | {"lit:raw/1B"}


def census_parts() -> list[np.ndarray]:
    """The form cases and the other zstd GPU tests' inputs (few long repeats) and the long-match cases."""
    return zf.form_parts() + gpu_inputs() + ldm_parts()


def test_census_covers_the_required_forms():
    """census_parts() reach every form _lzh requires, plus the block that is one span (no literals, one sequence)."""
    frames = [ldm.zstd_frame_lzl(p.tobytes()) for p in census_parts()]
    c = zf.census(frames)
    print("\nlzl census:")
    for name in sorted(c):
        print(f"  {name:24s} {c[name]:6d}{'  (required)' if name in REQUIRED_LZL else ''}")
    assert not REQUIRED_LZL - set(c), sorted(REQUIRED_LZL - set(c))
