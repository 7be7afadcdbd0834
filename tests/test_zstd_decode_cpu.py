"""The blob decoder's test set without a GPU: the fixture frames of tests/golden/zstd_frames.bin decode with libzstd
(pyarrow) to their seeded inputs, and the decoder's inputs -- the fixture, pyarrow's frames at levels -5, 1, 3, 9 and
19 on text, binary and repeated data, and this engine's frames (the restatements, byte-equal to the GPU's) -- reach
every form in zstd_dec_forms.REQUIRED_DECODE.  The C header's status values match the Python names."""
import re
from functools import lru_cache
from pathlib import Path

import numpy as np
import pytest

import zstd_dec_forms as zd
import zstd_forms as zf
import zstd_ent_ref as entref
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from pbs_plus_b200 import _lib

pa = pytest.importorskip("pyarrow")
ROOT = Path(__file__).resolve().parent.parent
LEVELS = (-5, 1, 3, 9, 19)


def corpora(n: int, seed: int):
    """The text, binary and repeated inputs the libzstd frames are made of."""
    return {"text": lzref.text_corpus(n, seed), "binary": hufref.binary_corpus(n, seed + 1),
            "repeated": np.tile(np.frombuffer(bytes(range(97)) * 3, np.uint8), n // 291 + 1)[:n]}


@lru_cache(maxsize=None)
def libzstd_payloads(n: int = 1 << 20, seed: int = 1):
    """(level, corpus name, payload, input) for every level and corpus"""
    out = []
    for lvl in LEVELS:
        codec = pa.Codec("zstd", compression_level=lvl)
        for name, data in corpora(n, seed).items():
            out.append((lvl, name, codec.compress(data.tobytes(), asbytes=True), data.tobytes()))
    return out


def engine_payloads():
    """_lz, _lze and _lzh frames of the form cases (the restatements; the GPU writes the same bytes)"""
    parts = [p for p, _ in zf.form_cases()[:6]]
    return [f(p.tobytes()) for f in (lzref.zstd_frame_lz, entref.zstd_frame_lze, hufref.zstd_frame_lzh) for p in parts]


def test_fixture_frames_decode_with_libzstd_to_their_seeded_inputs():
    cases = zd.fixture_cases()
    assert (zd.GOLDEN / "zstd_frames.bin").stat().st_size <= 1 << 20
    assert set(cases) == {"nofcs", "checksum_raw", "small_window", "ldm", "fcs_1", "fcs_2", "two_frames", "handmade"}
    for name, (payload, data) in cases.items():
        assert pa.decompress(payload, decompressed_size=len(data), codec="zstd", asbytes=True) == data, name


def test_the_decoder_test_set_reaches_every_required_form():
    payloads = [p for p, _ in zd.fixture_cases().values()]
    payloads += [p for _, _, p, _ in libzstd_payloads()]
    payloads += engine_payloads()
    c = zd.decode_census(payloads)
    print("\ndecoder census:")
    for form, k in sorted(c.items()):
        print(f"  {form:24s} {k}")
    missing = zd.REQUIRED_DECODE - set(c)
    assert not missing, missing


def test_frame_census_reads_each_frame_form():
    cases = zd.fixture_cases()
    assert zd.decode_census([cases["nofcs"][0]])["fcs:0"] >= 1
    two = zd.split_payload(cases["two_frames"][0])
    assert [k for k, _ in two] == ["zstd", "skippable", "zstd"]
    assert zd.frame_forms(two[2][1])[-1] == "checksum"
    assert "fcs:8" in zd.frame_forms(cases["handmade"][0])


def test_decode_status_values_match_the_header():
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    m = re.search(r"enum \{ (PBSGPU_DEC_OK = 0,[^}]*)\}", hdr)
    names = [x.strip().split()[0] for x in m.group(1).split(",")]
    assert names == ["PBSGPU_DEC_OK", "PBSGPU_DEC_BAD_MAGIC", "PBSGPU_DEC_BAD_CRC", "PBSGPU_DEC_ENCRYPTED",
                     "PBSGPU_DEC_BAD_FRAME", "PBSGPU_DEC_BAD_SIZE", "PBSGPU_DEC_BAD_CHECKSUM", "PBSGPU_DEC_BAD_DIGEST"]
    for k, name in enumerate(names):
        assert getattr(_lib, name[len("PBSGPU_"):]) == k
