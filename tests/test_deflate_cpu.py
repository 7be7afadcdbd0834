"""The Deflate restatement (tests/deflate_ref.py) on the CPU: every case decodes under zlib's raw inflate and under GNU
gzip's own inflate, every form and run-length code is reached (the test fails when one goes unreached), the lit/len
code's 15-bit and the code-length code's 7-bit limits are engaged, pieces joined with `more` give the one-piece stream,
and pbsgpu_crc32_combine and pbsgpu_deflate_bound hold."""
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import deflate_ref as dr
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from pbs_plus_b200 import engine

SEG = dr.SEGMENT


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=n, dtype=np.uint8).tobytes()


def skewed(n, seed, r=1.2):
    """Bytes with probabilities r^-rank over shuffled byte values: the unconstrained lit/len code wants more than 15
    bits, so the halving loop runs."""
    w = r ** -np.arange(256.0)
    p = w[np.random.default_rng(seed).permutation(256)]
    return np.random.default_rng(seed + 10).choice(256, size=n, p=p / p.sum()).astype(np.uint8).tobytes()


def cases():
    """name -> bytes: the sizes at every segment and stored-block edge, and zeros, random, text, binary data, all byte
    values, one byte value, repeats at distances 32768 and 32769, runs of 258 and 259, skewed symbol counts."""
    text = lzref.text_corpus(3 * SEG + 17, 3).tobytes()
    binary = hufref.binary_corpus(SEG + 4000, 4).tobytes()
    unit = rnd(32768, 5)
    out = {"empty": b"", "one": b"\x07", "three": b"abc", "four": b"abcd"}
    for n in (65535, 65536, SEG - 1, SEG, SEG + 1, 3 * SEG + 17):
        out[f"text_{n}"] = text[:n]
    for n in (65535, 65536, SEG + 1):
        out[f"random_{n}"] = rnd(n, n)
    out["zeros"] = bytes(2 * SEG + 5)
    out["binary"] = binary
    out["all_bytes"] = bytes(range(256)) * 300
    out["one_value"] = b"\x41" * 70000
    out["dist_32768"] = unit + unit[:5000] + rnd(100, 6)
    out["dist_32769"] = unit + b"\x00" + unit[:5000]
    out["run_258"] = rnd(50, 7) + b"\x55" * 259 + rnd(50, 8)
    out["run_259"] = rnd(50, 9) + b"\x55" * 260 + rnd(50, 10)
    out["skewed"] = skewed(SEG, 2)
    out["fibonacci"] = dr.fib_weighted(SEG)
    out["short_text"] = text[:300]
    return out


def gzip_member(stream: bytes, data: bytes) -> bytes:
    return (b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03" + stream + zlib.crc32(data).to_bytes(4, "little")
            + (len(data) & 0xFFFFFFFF).to_bytes(4, "little"))


@pytest.fixture(scope="module")
def streams():
    stats = {}
    out = {name: (data, dr.deflate(data, stats=stats)) for name, data in cases().items()}
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


def test_every_form_and_run_code_is_reached(streams):
    stats = streams[1]
    assert stats["forms"] == {"stored", "fixed", "dynamic"}, stats["forms"]
    assert stats["cl"] == {16, 17, 18}, stats["cl"]
    assert stats["maxbits"] == dr.LIT_MAXBITS
    assert stats["cl_maxbits"] == dr.CL_MAXBITS


def test_the_lit_len_limit_is_engaged():
    toks = dr.deflate_parse(cases()["skewed"])
    cnt = [0] * 286
    for t in toks:
        cnt[dr.len_code(t[0]) if isinstance(t, tuple) else t] += 1
    cnt[256] += 1
    assert max(dr.huffman_lengths(cnt, 99)) > dr.LIT_MAXBITS
    assert max(dr.huffman_lengths(cnt, dr.LIT_MAXBITS)) == dr.LIT_MAXBITS


def test_the_code_length_limit_is_engaged():
    toks = dr.deflate_parse(cases()["fibonacci"])
    runs = dr.dynamic_codes(toks)[4]
    cl = [0] * 19
    for s, _, _ in runs:
        cl[s] += 1
    assert max(dr.huffman_lengths(cl, 99)) > dr.CL_MAXBITS
    st = {}
    dr.deflate(cases()["fibonacci"], stats=st)
    assert st["forms"] == {"dynamic"} and st["cl_maxbits"] == dr.CL_MAXBITS


def test_huffman_lengths_halving_and_one_symbol():
    fib = [1, 1]
    while len(fib) < 19:
        fib.append(fib[-1] + fib[-2])
    assert max(dr.huffman_lengths(fib, 99)) == 18
    got = dr.huffman_lengths(fib, dr.CL_MAXBITS)
    assert max(got) == dr.CL_MAXBITS and sum(2.0 ** -x for x in got) <= 1
    assert dr.huffman_lengths([0, 5, 0], 15) == [0, 1, 0]


def test_parse_limits():
    toks = dr.deflate_parse(cases()["dist_32768"])
    assert any(isinstance(t, tuple) and t[1] == 32768 for t in toks)
    assert all(t[1] <= dr.WINDOW for t in toks if isinstance(t, tuple))
    assert not any(isinstance(t, tuple) and t[1] > dr.WINDOW for t in dr.deflate_parse(cases()["dist_32769"]))
    for name in ("run_258", "run_259", "zeros"):
        assert all(t[0] <= dr.MAX_MATCH for t in dr.deflate_parse(cases()[name]) if isinstance(t, tuple))


def test_pieces_join_to_the_one_piece_stream():
    data = lzref.text_corpus(3 * SEG + 17, 3).tobytes()
    whole = dr.deflate(data)
    for cuts in ([SEG], [SEG, 3 * SEG], [2 * SEG, 3 * SEG]):
        parts, lo = [], 0
        for c in cuts:
            parts.append(dr.deflate(data[lo:c], more=True))
            lo = c
        parts.append(dr.deflate(data[lo:]))
        assert b"".join(parts) == whole
    assert dr.deflate(b"", more=True) == b"" and dr.deflate(b"") == b"\x03\x00"


def test_crc32_combine_matches_zlib():
    rng = np.random.default_rng(11)
    for la, lb in ((0, 0), (0, 5), (7, 0), (1, 1), (1000, 131072), (5 << 20, 3)):
        a, b = rnd(la, la + 1), rnd(lb, lb + 2)
        assert engine.crc32_combine(zlib.crc32(a), zlib.crc32(b), lb) == zlib.crc32(a + b)
    # lengths beyond 4 GiB: combining zeros twice equals combining once with the sum
    c = int(rng.integers(0, 1 << 32))
    z = zlib.crc32(bytes(1 << 20))
    step = engine.crc32_combine(engine.crc32_combine(c, z, 1 << 20), z, 1 << 20)
    assert step == engine.crc32_combine(c, zlib.crc32(bytes(2 << 20)), 2 << 20)


def test_bound_on_incompressible_data():
    for n in (1, 65535, SEG, SEG + 1, 2 * SEG + 65536):
        data = rnd(n, n + 3)
        assert len(dr.deflate(data)) <= engine.deflate_bound(n)
