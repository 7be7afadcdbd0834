"""The Deflate chain-parse restatement (tests/deflate_chain_ref.py) on the CPU: every case inflates under zlib and GNU
gzip and stays within pbsgpu_deflate_bound; offsets reach exactly 32768 and no further, matches stop at 258 bytes and at
the segment's end and overlap their source; 3-byte matches are taken, near and far; a segment
takes at most LZ_MAX_SEQ matches; pieces joined with `more` give the one-call stream; the parse takes a lazy step in
some case and the margin refuses one in another; and the chosen constants are pinned against the greedy stream and
zlib per 128 KiB segment (DESIGN.md K16d)."""
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import deflate_chain_ref as ch
import deflate_ref as dr
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from pbs_plus_b200 import engine

SEG = dr.SEGMENT


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=n, dtype=np.uint8).tobytes()


def three_byte_words(n, seed, vocab=64, junk=1):
    """3-byte words drawn from a small vocabulary, each followed by `junk` random bytes: most matches are exactly 3
    bytes long, near ones (and far ones in a long segment)."""
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 256, (vocab, 3), dtype=np.uint8)
    out = np.concatenate([words[rng.integers(0, vocab, n // (3 + junk) + 1)],
                          rng.integers(0, 256, (n // (3 + junk) + 1, junk), dtype=np.uint8)], axis=1)
    return out.reshape(-1)[:n].tobytes()


def seq_cap_segment(seed=41):
    """A segment whose parse would take more than LZ_MAX_SEQ matches: 3-byte words from 16 with no bytes between,
    so matches are short and back to back."""
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 256, (4096, 3), dtype=np.uint8)
    return words[rng.integers(0, 4096, SEG // 3 + 1)].reshape(-1)[:SEG].tobytes()


def cases():
    """name -> bytes: tiny, off-grid, constant and half-constant inputs, the window and length edges, overlapping
    sources, matches ending at a segment's end, 3-byte matches and a segment past the sequence cap."""
    text = lzref.text_corpus(3 * SEG + 17, 3).tobytes()
    unit = rnd(32768, 5)
    tail = rnd(SEG - 700, 6)
    out = {"empty": b"", "one": b"\x07", "two": b"\x07\x07", "three": b"abc", "four": b"abab"}
    for n in (SEG - 1, SEG, SEG + 1, 3 * SEG + 17):
        out[f"text_{n}"] = text[:n]
    out["zeros"] = bytes(2 * SEG + 5)
    out["one_value"] = b"\x41" * 70000
    out["half_zero"] = (bytes(SEG // 2) + rnd(SEG, 7) + bytes(SEG // 2))
    out["binary"] = hufref.binary_corpus(SEG + 4000, 4).tobytes()
    out["random"] = rnd(SEG + 1, 8)
    out["dist_32768"] = unit + unit[:5000] + rnd(100, 9)
    out["dist_32769"] = unit + b"\x00" + unit[:5000]
    out["run_258"] = rnd(50, 10) + b"\x55" * 259 + rnd(50, 11)
    out["run_259"] = rnd(50, 12) + b"\x55" * 260 + rnd(50, 13)
    out["overlap"] = b"".join(rnd(300, 20 + p) + rnd(p, 30 + p) * (3000 // p) for p in (1, 2, 3, 5, 7))
    out["ends_at_segment_end"] = tail + tail[-20000:-19300] + text[:SEG // 2]   # a 700-byte match ends at byte SEG
    out["ends_at_stream_end"] = rnd(5000, 14) + rnd(5000, 14)[:777]
    out["three_byte_near"] = three_byte_words(3 * SEG, 15)
    out["three_byte_far"] = three_byte_words(SEG, 16, vocab=4000)
    out["seq_cap"] = seq_cap_segment() + text[:1000]
    return out


def gzip_member(stream: bytes, data: bytes) -> bytes:
    return (b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03" + stream + zlib.crc32(data).to_bytes(4, "little")
            + (len(data) & 0xFFFFFFFF).to_bytes(4, "little"))


def matches(data: bytes):
    """[(segment, position in segment, length, offset)] of the chain parse of `data`."""
    d = bytes(data)
    L, O = (x.tolist() for x in ch.best_all(d)[ch.DCH_DEPTH])
    out = []
    for k in range((len(d) + SEG - 1) // SEG):
        lo, hi = k * SEG, min(len(d), (k + 1) * SEG)
        out += [(k, m - lo, l, o) for m, l, o in ch.parse(L, O, lo, hi)]
    return out


@pytest.fixture(scope="module")
def streams():
    stats = {}
    out = {name: (data, ch.deflate(data, stats=stats)) for name, data in cases().items()}
    return out, stats


def test_every_case_inflates_under_zlib(streams):
    for name, (data, s) in streams[0].items():
        assert zlib.decompress(s, -15) == data, name
        assert len(s) <= dr.bound(len(data)) == engine.deflate_bound(len(data)), name


@pytest.mark.skipif(shutil.which("gzip") is None, reason="GNU gzip is not installed")
def test_every_case_inflates_under_gzip(streams):
    for name, (data, s) in streams[0].items():
        r = subprocess.run(["gzip", "-dc"], input=gzip_member(s, data), capture_output=True)
        assert r.returncode == 0 and r.stdout == data, (name, r.stderr)


def test_the_segment_format_is_deflate_refs(streams):
    """What the parse does not decide is the greedy stream's: the empty stream, tiny inputs and incompressible data."""
    for name in ("empty", "one", "two", "three", "random"):
        data, s = streams[0][name]
        assert s == dr.deflate(data), name
    assert streams[1]["forms"] == {"stored", "fixed", "dynamic"}


def test_window_and_length_limits():
    cs = cases()
    assert any(o == 32768 for _, _, _, o in matches(cs["dist_32768"]))
    assert all(o <= ch.WINDOW for _, _, _, o in matches(cs["dist_32769"]))
    assert not any(L > 16 for _, _, L, _ in matches(cs["dist_32769"]))   # the copy 32769 back is out of reach
    for name in ("run_258", "run_259", "zeros", "one_value"):
        ms = matches(cs[name])
        assert all(L <= ch.MAX_MATCH for _, _, L, _ in ms) and any(L == ch.MAX_MATCH for _, _, L, _ in ms), name
    assert any(L == 258 and o == 1 for _, _, L, o in matches(cs["run_259"]))


def test_overlapping_sources_and_segment_ends():
    cs = cases()
    ms = matches(cs["overlap"])
    assert {o for _, _, _, o in ms if o < 8} >= {1, 2, 3, 5, 7}
    assert any(L > o for _, _, L, o in ms)   # the source overlaps the match
    ends = [(k, m + L) for k, m, L, _ in matches(cs["ends_at_segment_end"])]
    assert (0, SEG) in ends and all(e <= SEG for k, e in ends if k == 0)
    d = cs["ends_at_stream_end"]
    assert any(m + L == len(d) for _, m, L, _ in matches(d))


def test_three_byte_matches_near_and_far():
    cs = cases()
    assert ch.DCH_MINMATCH == 3
    near = [o for _, _, L, o in matches(cs["three_byte_near"]) if L == 3]
    far = [o for _, _, L, o in matches(cs["three_byte_far"]) if L == 3]
    assert near and min(near) < 64
    assert far and max(far) > 4096   # no zlib-like TOO_FAR rule: the sweep found it does not pay


def test_a_segment_takes_at_most_lz_max_seq_matches():
    d = cases()["seq_cap"]
    L, O = (x.tolist() for x in ch.best_all(d)[ch.DCH_DEPTH])
    seqs = ch.parse(L, O, 0, SEG)
    assert len(seqs) == ch.LZ_MAX_SEQ
    end = seqs[-1][0] + seqs[-1][1]
    assert any(L[end:SEG])   # matches were left: the rest of the segment went out as literals


def test_lazy_steps_are_taken_and_refused(streams):
    stats = streams[1]
    assert stats.get("lazy", 0) > 0, "no lazy step was taken"
    assert stats.get("refused", 0) > 0, "the margin refused no lazy step"
    # the margin decides some step: without it the parse of the text case moves on more often
    d = cases()["text_393233"]
    s0, s4 = {}, {}
    ch.deflate(d, stats=s0, margin=0)
    ch.deflate(d, stats=s4)
    assert s0["lazy"] > s4["lazy"]


def test_pieces_join_to_the_one_piece_stream():
    data = lzref.text_corpus(3 * SEG + 17, 3).tobytes()
    whole = ch.deflate(data)
    for cuts in ([SEG], [SEG, 3 * SEG], [2 * SEG, 3 * SEG]):
        parts, lo = [], 0
        for c in cuts:
            parts.append(ch.deflate(data[lo:c], more=True))
            lo = c
        parts.append(ch.deflate(data[lo:]))
        assert b"".join(parts) == whole
    assert ch.deflate(b"", more=True) == b"" and ch.deflate(b"") == b"\x03\x00"


def zlib_per_segment(d: bytes, level: int) -> int:
    tot = 0
    for k in range(0, len(d), SEG):
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        tot += len(c.compress(d[k:k + SEG]) + c.flush())
    return tot


@pytest.mark.parametrize("mib", [1, 8])
@pytest.mark.parametrize("corpus", ["text", "binary"])
def test_the_constants_meet_the_sweep_rule(corpus, mib):
    """DESIGN.md K16d: no row with DEPTH <= 32 reaches zlib -4 per segment on the binary corpus, so the constants are
    the best row, (MINMATCH 3, DEPTH 32, LAZY 2, MARGIN 4).  Pinned: smaller than the greedy stream; on text at or
    below zlib -4 per segment; on binary at most zlib -1 per segment at 8 MiB and within 0.2 % of it at 1 MiB (zlib
    starts a new block with new codes every 16 K symbols, K15 writes one per segment)."""
    assert (ch.DCH_MINMATCH, ch.DCH_DEPTH, ch.DCH_LAZY, ch.DCH_MARGIN) == (3, 32, 2, 4)
    d = bytes(lzref.text_corpus(mib << 20, 1) if corpus == "text" else hufref.binary_corpus(mib << 20, 2))
    s = len(ch.deflate(d))
    assert s < len(dr.deflate(d))
    if corpus == "text":
        assert s <= zlib_per_segment(d, 4)
    else:
        assert s <= zlib_per_segment(d, 1) * (1.002 if mib == 1 else 1)
