"""Writes tests/golden/zstd_frames.bin (the payloads back to back) and tests/golden/zstd_frames.json (per case: offset
and length of its payload, the recipe of its input and the input's SHA-256): zstd payloads for the blob decoder's
tests in forms pyarrow's one-shot encoder does not write.  Run once, with a system libzstd (ctypes,
ZSTD_compressStream2), from the repository root:

    python tests/golden/make_zstd_frames.py

Inputs are rebuilt from their recipes (tests/zstd_dec_forms.decode_input: seeded parts), so no input bytes are stored.
The cases:
  nofcs          streamed in 16 KiB pieces with the content size unknown: windowed frames without Frame_Content_Size
  checksum_raw   checksumFlag=1 and windowLog=10 (1 KiB blocks) over text, 3 KiB of random bytes (Raw_Blocks) and
                 text; the decoder tests flip a byte inside a Raw_Block of it for BAD_CHECKSUM
  small_window   windowLog=10: 1 KiB blocks, dozens of them
  ldm            long-distance matching on (windowLog=24), input repeating 4 KiB of random bytes 30 KB later
  two_frames     two frames with a skippable frame between them, the second with checksumFlag=1
  fcs_1, fcs_2   short single-segment frames with a 1- and a 2-byte Frame_Content_Size
  handmade       assembled here from RFC 8878: one frame with an 8-byte Frame_Content_Size and a Dictionary_ID field of
                 zero, whose Compressed_Blocks have no sequences and RLE literals (1- and 3-byte headers) or raw
                 literals with a 1-byte header, next to an RLE_Block and a Raw_Block.  libzstd writes none of these
                 literal forms on the corpora above, so they are built by hand.
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
import hashlib
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
from zstd_dec_forms import decode_input  # noqa: E402

OUT = ROOT / "tests" / "golden" / "zstd_frames"

# ZSTD_cParameter values (zstd.h, stable API)
C_LEVEL, C_WINDOWLOG, C_LDM = 100, 101, 160
C_CONTENTSIZE, C_CHECKSUM = 200, 201
E_CONTINUE, E_END = 0, 2


class InBuf(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class OutBuf(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


def _lib():
    L = C.CDLL(ctypes.util.find_library("zstd") or "libzstd.so.1")
    L.ZSTD_createCCtx.restype = C.c_void_p
    L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
    L.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.ZSTD_CCtx_setParameter.restype = C.c_size_t
    L.ZSTD_compressStream2.argtypes = [C.c_void_p, C.POINTER(OutBuf), C.POINTER(InBuf), C.c_int]
    L.ZSTD_compressStream2.restype = C.c_size_t
    L.ZSTD_isError.argtypes = [C.c_size_t]
    L.ZSTD_versionString.restype = C.c_char_p
    return L


def compress(L, data: bytes, params: dict, piece: int | None = None) -> bytes:
    """One frame of `data` through ZSTD_compressStream2; `piece`: fed in pieces, so the content size stays unknown."""
    cctx = L.ZSTD_createCCtx()
    try:
        for k, v in params.items():
            assert not L.ZSTD_isError(L.ZSTD_CCtx_setParameter(cctx, k, v))
        src = C.create_string_buffer(data, len(data))
        cap = len(data) + (len(data) >> 7) + 4096
        dst = C.create_string_buffer(cap)
        out = OutBuf(C.addressof(dst), cap, 0)
        step = piece or max(1, len(data))
        for lo in range(0, max(1, len(data)), step):
            hi = min(len(data), lo + step)
            inb = InBuf(C.addressof(src) + lo, hi - lo, 0)
            mode = E_END if hi == len(data) else E_CONTINUE
            while True:
                rem = L.ZSTD_compressStream2(cctx, C.byref(out), C.byref(inb), mode)
                assert not L.ZSTD_isError(rem)
                if (mode == E_END and rem == 0) or (mode == E_CONTINUE and inb.pos == inb.size):
                    break
        return dst.raw[:out.pos]
    finally:
        L.ZSTD_freeCCtx(cctx)


def handmade(data: bytes) -> bytes:
    """The `handmade` frame (see the module docstring) of data = decode_input(HANDMADE)."""
    def block(content: bytes, btype: int, size: int, last: bool) -> bytes:
        return (int(last) | btype << 1 | size << 3).to_bytes(3, "little") + content

    parts = [
        block(bytes([20 << 3 | 1, ord("a")]) + b"\0", 2, 3, False),                          # RLE literals, 1-byte header
        block(bytes([(5000 & 15) << 4 | 3 << 2 | 1, (5000 >> 4) & 255, 5000 >> 12, ord("b")]) + b"\0", 2, 5, False),
        block(bytes([24 << 3]) + bytes(range(24)) + b"\0", 2, 26, False),                  # raw literals, 1-byte header
        block(bytes([ord("c")]), 1, 3000, False),                                          # RLE_Block
        block(b"raw block bytes", 0, 15, True),                                            # Raw_Block
    ]
    fhd = 3 << 6 | 1 << 5 | 1                                   # 8-byte FCS, single segment, 1-byte Dictionary_ID
    frame = (0xFD2FB528).to_bytes(4, "little") + bytes([fhd, 0]) + len(data).to_bytes(8, "little") + b"".join(parts)
    return frame


# the handmade frame's content
HANDMADE = [["byte", ord("a"), 20], ["byte", ord("b"), 5000], ["hex", bytes(range(24)).hex(), 0], ["byte", ord("c"), 3000],
            ["hex", b"raw block bytes".hex(), 0]]


def main():
    L = _lib()
    cases = {
        "nofcs": ([["text", 11, 30_000]], lambda d: compress(L, d, {C_LEVEL: 3, C_CONTENTSIZE: 0}, piece=16 << 10)),
        "checksum_raw": ([["text", 12, 12_000], ["random", 13, 3 << 10], ["text", 14, 6_000]],
                         lambda d: compress(L, d, {C_LEVEL: 3, C_CHECKSUM: 1, C_WINDOWLOG: 10})),
        "small_window": ([["text", 15, 20_000]], lambda d: compress(L, d, {C_LEVEL: 5, C_WINDOWLOG: 10})),
        "ldm": ([["random", 16, 4 << 10], ["text", 17, 30_000], ["copy", 30_000 + (4 << 10), 4 << 10]],
                lambda d: compress(L, d, {C_LEVEL: 3, C_LDM: 1, C_WINDOWLOG: 24})),
        "fcs_1": ([["text", 18, 200]], lambda d: compress(L, d, {C_LEVEL: 3})),
        "fcs_2": ([["text", 19, 3_000]], lambda d: compress(L, d, {C_LEVEL: 3})),
    }
    meta = {"libzstd": L.ZSTD_versionString().decode(), "cases": {}}
    blob = bytearray()

    def put(name, recipe, payload):
        data = decode_input(recipe).tobytes()
        meta["cases"][name] = {"recipe": recipe, "sha256": hashlib.sha256(data).hexdigest(), "offset": len(blob),
                               "length": len(payload)}
        blob.extend(payload)

    for name, (recipe, fn) in cases.items():
        put(name, recipe, fn(decode_input(recipe).tobytes()))
    a, b = [["binary", 20, 15_000]], [["text", 21, 10_000]]
    skip = (0x184D2A53).to_bytes(4, "little") + (11).to_bytes(4, "little") + b"not content"
    fa = compress(L, decode_input(a).tobytes(), {C_LEVEL: 1})
    fb = compress(L, decode_input(b).tobytes(), {C_LEVEL: 6, C_CHECKSUM: 1})
    put("two_frames", a + b, fa + skip + fb)
    put("handmade", HANDMADE, handmade(decode_input(HANDMADE).tobytes()))
    OUT.with_suffix(".bin").write_bytes(bytes(blob))
    OUT.with_suffix(".json").write_text(json.dumps(meta, indent=1) + "\n")
    print(OUT, len(blob), "bytes of payloads")


if __name__ == "__main__":
    main()
