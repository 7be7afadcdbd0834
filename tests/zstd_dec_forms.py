"""Which frame forms the blob decoder's inputs reach (pbsgpu_blob_decode_batch), on top of zstd_forms' block census, and
the decoder's fixture (tests/golden/zstd_frames.json and .bin, written by tests/golden/make_zstd_frames.py).  Test
infrastructure for tests/test_zstd_decode_cpu.py and tests/test_gpu_blob_decode.py."""
from __future__ import annotations

import hashlib
import json
from collections import Counter
from pathlib import Path

import numpy as np

from zstd_forms import ZSTD_MAGIC, census
from zstd_lz_ref import text_corpus

GOLDEN = Path(__file__).resolve().parent / "golden"


# A compressed DataBlob's payload is one or more frames with skippable frames allowed between them.  Frame form names:
#   frame:single | frame:windowed      Single_Segment_Flag
#   fcs:0 | fcs:1 | fcs:2 | fcs:4 | fcs:8   Frame_Content_Size field size (0: absent)
#   checksum                           Content_Checksum_Flag
#   skippable | multi-frame            a skippable frame; more than one zstd frame in a payload
SKIPPABLE_MASK, SKIPPABLE_MAGIC = 0xFFFFFFF0, 0x184D2A50


def frame_end(data: bytes, pos: int) -> int:
    """End of the zstd frame that starts at `pos` (its blocks walked by their headers)."""
    fhd = data[pos + 4]
    single, checksum, did = (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
    p = pos + 5 + (not single) + (0, 1, 2, 4)[did] + ((1 if single else 0), 2, 4, 8)[fhd >> 6]
    while True:
        h = int.from_bytes(data[p:p + 3], "little")
        p += 3 + (1 if (h >> 1) & 3 == 1 else h >> 3)
        if h & 1:
            return p + 4 * checksum


def split_payload(data: bytes) -> list[tuple[str, bytes]]:
    """The frames of a payload in order: ("zstd", frame) or ("skippable", frame)."""
    data, out, pos = bytes(data), [], 0
    while pos < len(data):
        magic = int.from_bytes(data[pos:pos + 4], "little")
        if magic & SKIPPABLE_MASK == SKIPPABLE_MAGIC:
            end = pos + 8 + int.from_bytes(data[pos + 4:pos + 8], "little")
            out.append(("skippable", data[pos:end]))
        elif magic == ZSTD_MAGIC:
            end = frame_end(data, pos)
            out.append(("zstd", data[pos:end]))
        else:
            raise ValueError("neither a zstd nor a skippable frame")
        pos = end
    return out


def frame_forms(frame: bytes) -> list[str]:
    """The named frame forms of one zstd frame."""
    fhd = frame[4]
    single = (fhd >> 5) & 1
    fcs = ((1 if single else 0), 2, 4, 8)[fhd >> 6]
    out = ["frame:single" if single else "frame:windowed", f"fcs:{fcs}"]
    if (fhd >> 2) & 1:
        out.append("checksum")
    return out


def decode_census(payloads) -> Counter:
    """Frame and block forms over blob payloads (census() plus frame_forms, skippable and multi-frame)."""
    c = Counter()
    for pl in payloads:
        frames = split_payload(pl)
        if sum(kind == "zstd" for kind, _ in frames) > 1:
            c["multi-frame"] += 1
        for kind, fr in frames:
            if kind == "skippable":
                c["skippable"] += 1
                continue
            c.update(frame_forms(fr))
            c.update(census([fr]))
    return c


# The forms the decoder's tests must reach (tests/test_zstd_decode_cpu.py checks the set, the GPU tests decode it)
REQUIRED_DECODE = {
    "block:raw", "block:rle", "block:compressed",
    "lit:raw/1B", "lit:raw/2B", "lit:raw/3B", "lit:rle/1B", "lit:rle/3B",
    "lit:huf/sf0", "lit:huf/sf1", "lit:huf/sf2", "lit:huf/sf3",
    "lit:treeless/sf0", "lit:treeless/sf1", "lit:treeless/sf2",
    "tree:direct", "tree:fse/log5/odd", "tree:fse/log5/even",
    "nseq:0", "nseq:1B", "nseq:2B", "nseq:3B", "tree:fse/log6/odd",
    "modes:PPP", "modes:FFF", "modes:FFX", "modes:XXX", "modes:PFF", "modes:PXX", "modes:XXR", "modes:PRP",
    "frame:single", "frame:windowed", "fcs:0", "fcs:1", "fcs:2", "fcs:4", "fcs:8",
    "checksum", "skippable", "multi-frame",
}


def decode_input(parts) -> np.ndarray:
    """The input of a decoder fixture case from its recipe: parts [kind, seed_or_distance, n] concatenated, kind one of
    "text" (zstd_lz_ref.text_corpus), "binary" (zstd_huf_ref.binary_corpus), "random" (uniform bytes), "byte" (n copies
    of the byte `seed`), "hex" (the bytes `seed` spells in hex) and "copy" (the n bytes that start `seed` bytes back)."""
    from zstd_huf_ref import binary_corpus
    out = bytearray()
    for kind, s, n in parts:
        if kind == "text":
            out += text_corpus(n, s).tobytes()
        elif kind == "binary":
            out += binary_corpus(n, s).tobytes()
        elif kind == "random":
            out += np.random.default_rng(s).integers(0, 256, n, dtype=np.uint8).tobytes()
        elif kind == "byte":
            out += bytes([s]) * n
        elif kind == "hex":
            out += bytes.fromhex(s)
        elif kind == "copy":
            start = len(out) - s
            out += out[start:start + n]
        else:
            raise ValueError(kind)
    return np.frombuffer(bytes(out), np.uint8)


def fixture_cases() -> dict[str, tuple[bytes, bytes]]:
    """name -> (payload, input) of the decoder's fixture; each input is rebuilt from its recipe and checked against its
    SHA-256."""
    meta = json.loads((GOLDEN / "zstd_frames.json").read_text())
    blob = (GOLDEN / "zstd_frames.bin").read_bytes()
    out = {}
    for name, c in meta["cases"].items():
        data = decode_input(c["recipe"]).tobytes()
        assert hashlib.sha256(data).hexdigest() == c["sha256"], name
        out[name] = (blob[c["offset"]:c["offset"] + c["length"]], data)
    return out
