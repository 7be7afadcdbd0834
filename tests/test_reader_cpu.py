"""The archive reader without a GPU: its declarations are in the header, and the statuses and flag it adds have the
values the bindings use."""
import re
from pathlib import Path

from pbs_plus_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent


def test_reader_is_declared():
    hdr = " ".join((ROOT / "include" / "pbsgpu.h").read_text().split())
    assert "typedef struct pbsgpu_reader pbsgpu_reader;" in hdr
    for name in ("pbsgpu_reader_open", "pbsgpu_reader_close", "pbsgpu_reader_size", "pbsgpu_reader_plan", "pbsgpu_reader_read"):
        assert re.search(rf"\b{name}\(", hdr) and name in _lib.SYMBOLS, name
    assert "int pbsgpu_reader_open(pbsgpu_ctx *ctx, const uint8_t *didx, uint64_t size, const pbsgpu_crypt *crypt, " \
           "uint64_t cache_bytes, pbsgpu_reader **out);" in hdr


def test_missing_and_bad_header_follow_the_decode_statuses():
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    assert re.search(r"enum \{ PBSGPU_DEC_MISSING = PBSGPU_DEC_BAD_TAG \+ 1,.*?\n\s*PBSGPU_DEC_BAD_HEADER \};", hdr, re.S)
    assert _lib.DEC_MISSING == _lib.DEC_BAD_TAG + 1 == 9
    assert _lib.DEC_BAD_HEADER == _lib.DEC_MISSING + 1 == 10


def test_read_payload_flag():
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    assert re.search(r"#define PBSGPU_READ_PAYLOAD 1u\b", hdr)
    assert _lib.READ_PAYLOAD == 1
