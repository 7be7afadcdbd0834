"""The zstd decoder upstream restores chunks with, as a test reference: `zstd::stream::decode_all` drives libzstd's
streaming decoder, `ZSTD_decompressStream`, with default parameters.  It is called here through ctypes on the system
`libzstd.so.1`.  Test infrastructure for tests/test_zstd_edges_cpu.py and the GPU decode tests.

libzstd's one-shot entry point (`ZSTD_decompress`, which pyarrow's `decompress` calls) reads frames the streaming
decoder refuses: the streaming decoder's default `windowLogMax` is 27, so a frame whose Window_Size is above 2^27 + 1
bytes fails with "Frame requires too much memory for decoding", while the one-shot call decodes it.

The output buffer is a fixed 4 KiB.  When a frame states its Frame_Content_Size, the whole frame is in the input, and
the output space is at least that size, ZSTD_decompressStream decodes the frame in one step and skips the window
check.  With 4 KiB of output that shortcut applies only to frames whose content is at most 4 KiB, so a frame that is to
test the window limit has no Frame_Content_Size, or one above 4 KiB."""
from __future__ import annotations

import ctypes
from functools import lru_cache

import pytest

OUT_BUF = 4096


class _Buf(ctypes.Structure):       # ZSTD_inBuffer and ZSTD_outBuffer have the same layout
    _fields_ = [("ptr", ctypes.c_void_p), ("size", ctypes.c_size_t), ("pos", ctypes.c_size_t)]


@lru_cache(maxsize=1)
def _lib():
    try:
        L = ctypes.CDLL("libzstd.so.1")
    except OSError:
        return None
    L.ZSTD_createDStream.restype = ctypes.c_void_p
    L.ZSTD_freeDStream.argtypes = [ctypes.c_void_p]
    L.ZSTD_initDStream.argtypes = [ctypes.c_void_p]
    L.ZSTD_initDStream.restype = ctypes.c_size_t
    L.ZSTD_decompressStream.argtypes = [ctypes.c_void_p, ctypes.POINTER(_Buf), ctypes.POINTER(_Buf)]
    L.ZSTD_decompressStream.restype = ctypes.c_size_t
    L.ZSTD_isError.argtypes = [ctypes.c_size_t]
    L.ZSTD_isError.restype = ctypes.c_uint
    L.ZSTD_getErrorName.argtypes = [ctypes.c_size_t]
    L.ZSTD_getErrorName.restype = ctypes.c_char_p
    L.ZSTD_versionString.restype = ctypes.c_char_p
    return L


def available() -> bool:
    return _lib() is not None


def require():
    """Skips the calling test when the system libzstd is missing."""
    if not available():
        pytest.skip("libzstd.so.1 (the streaming reference decoder) is not installed")


def version() -> str:
    return _lib().ZSTD_versionString().decode()


def stream_decode(payload: bytes) -> bytes | str:
    """The frames of `payload` decoded as `zstd::stream::decode_all` does: every frame (skippable ones skipped) until the
    input ends.  Returns the content, or libzstd's error name; input that ends inside a frame gives "incomplete frame"."""
    L = _lib()
    if L is None:
        raise RuntimeError("libzstd.so.1 is not installed")
    src = ctypes.create_string_buffer(bytes(payload), len(payload) or 1)
    dst = ctypes.create_string_buffer(OUT_BUF)
    ds = L.ZSTD_createDStream()
    try:
        r = L.ZSTD_initDStream(ds)
        if L.ZSTD_isError(r):
            return L.ZSTD_getErrorName(r).decode()
        inb = _Buf(ctypes.cast(src, ctypes.c_void_p), len(payload), 0)
        out = bytearray()
        while True:   # until the input is used up and the last frame is complete, or no call makes progress
            outb = _Buf(ctypes.cast(dst, ctypes.c_void_p), OUT_BUF, 0)
            before = inb.pos
            hint = L.ZSTD_decompressStream(ds, ctypes.byref(outb), ctypes.byref(inb))
            if L.ZSTD_isError(hint):
                return L.ZSTD_getErrorName(hint).decode()
            out += dst.raw[:outb.pos]
            if inb.pos == inb.size and hint == 0:
                return bytes(out)
            if inb.pos == inb.size and inb.pos == before and outb.pos == 0:
                return "incomplete frame"
    finally:
        L.ZSTD_freeDStream(ds)
