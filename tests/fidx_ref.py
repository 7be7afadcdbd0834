"""Restatement of the PBS fixed index (.fidx) for the tests: upstream pbs-datastore fixed_index.rs, restated here
(UNVERIFIED against the Go module, as the .didx restatement in oracle/pyref.py is).  Never imported by the product.

Header (4096 bytes): magic[8], uuid[16], ctime i64 LE, index_csum[32] = SHA-256 over the digest table, size u64 LE
(image bytes), chunk_size u64 LE, zero padding.  Body: ceil(size / chunk_size) digests of 32 bytes; chunk i covers
[i * chunk_size, min((i + 1) * chunk_size, size)).
"""
from __future__ import annotations

import hashlib

FIDX_LABEL = b"Proxmox Backup fixed sized chunk index v1.0"
FIDX_MAGIC = bytes([0x2f, 0x7f, 0x41, 0xed, 0x91, 0xfd, 0x0f, 0xcd])


def n_chunks(size: int, chunk_size: int) -> int:
    return -(-size // chunk_size)


def chunk_digests(image: bytes, chunk_size: int, key: bytes | None = None) -> list[bytes]:
    """SHA-256 of every fixed chunk; with `key` (an id_key) the keyed digest SHA-256(chunk || key)."""
    return [hashlib.sha256(image[i:i + chunk_size] + (key or b"")).digest() for i in range(0, len(image), chunk_size)]


def fidx_build(digests, size: int, chunk_size: int, uuid: bytes = b"\0" * 16, ctime: int = 0) -> bytes:
    body = b"".join(bytes(d) for d in digests)
    assert len(body) == 32 * n_chunks(size, chunk_size)
    hdr = bytearray(4096)
    hdr[0:8] = FIDX_MAGIC
    hdr[8:24] = bytes(uuid).ljust(16, b"\0")[:16]
    hdr[24:32] = int(ctime).to_bytes(8, "little", signed=True)
    hdr[32:64] = hashlib.sha256(body).digest()
    hdr[64:72] = int(size).to_bytes(8, "little")
    hdr[72:80] = int(chunk_size).to_bytes(8, "little")
    return bytes(hdr) + body


def fidx_parse(image: bytes, verify: bool = True):
    """-> (size, chunk_size, [digest]); ValueError for what the library rejects with EINVAL."""
    image = bytes(image)
    if len(image) < 4096 or image[:8] != FIDX_MAGIC:
        raise ValueError("not a fixed index image")
    size = int.from_bytes(image[64:72], "little")
    cs = int.from_bytes(image[72:80], "little")
    if cs == 0 or cs >= 1 << 32:
        raise ValueError("chunk_size out of range")
    n = n_chunks(size, cs)
    if len(image) != 4096 + 32 * n:
        raise ValueError("length does not match size and chunk_size")
    body = image[4096:]
    if verify and hashlib.sha256(body).digest() != image[32:64]:
        raise ValueError("index checksum mismatch")
    return size, cs, [body[32 * i:32 * i + 32] for i in range(n)]
