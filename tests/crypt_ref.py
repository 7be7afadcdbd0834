"""Restatement of PBS encrypt mode for the tests (upstream pbs-tools crypt_config.rs, pbs-datastore data_blob.rs and
file_formats.rs; the module source is absent here, so every constant is UNVERIFIED-HERE like the other format
constants).  It uses `cryptography`'s AESGCM, hashlib's PBKDF2 and SHA-256 and the zstd restatements, so nothing in it
depends on the product's AES.

- CryptConfig::new(enc_key): id_key = PBKDF2-HMAC-SHA256(password=enc_key, salt=b"_id_key", iterations=10, dklen=32).
- compute_digest(data) = SHA-256(data || id_key): the key at the end, against length extension.
- Encrypted blob = { magic[8], crc32 LE, iv[16], tag[16], ciphertext }: AES-256-GCM under enc_key with the 16-byte IV
  (GCM's non-96-bit IV path) and empty AAD; the CRC covers the ciphertext only (compute_crc skips the 44-byte header).
- Compress, then encrypt: the zstd frame is encrypted when it is smaller than the chunk, else the raw chunk.
"""
from __future__ import annotations

import hashlib
import zlib

from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
from cryptography.hazmat.primitives.ciphers.aead import AESGCM

from oracle import pyref
import zstd_ent_ref as entref
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref

ENCRYPTED_BLOB_MAGIC_1_0 = bytes([0x7b, 0x67, 0x85, 0xbe, 0x22, 0x2d, 0x4c, 0xf0])
ENCR_COMPR_BLOB_MAGIC_1_0 = bytes([0xe6, 0x59, 0x1b, 0xbf, 0x0b, 0xbf, 0xd8, 0x0b])
MAGIC_LABELS = {
    ENCRYPTED_BLOB_MAGIC_1_0: "Proxmox Backup encrypted blob v1.0",
    ENCR_COMPR_BLOB_MAGIC_1_0: "Proxmox Backup zstd compressed encrypted blob v1.0",
}
HEADER = 44

# the frame builder of each blob mode of the product (None: the payload is always the raw chunk)
FRAMES = {"raw": None, "z": pyref.zstd_frame_rle_raw, "lz": lzref.zstd_frame_lz, "lze": entref.zstd_frame_lze,
          "lzh": hufref.zstd_frame_lzh}


def id_key(enc_key: bytes) -> bytes:
    return hashlib.pbkdf2_hmac("sha256", bytes(enc_key), b"_id_key", 10, 32)


def compute_digest(data: bytes, ident: bytes) -> bytes:
    return hashlib.sha256(bytes(data) + bytes(ident)).digest()


def gcm_encrypt(key: bytes, iv: bytes, data: bytes) -> tuple[bytes, bytes]:
    """(ciphertext, tag) of AES-256-GCM with empty AAD."""
    out = AESGCM(bytes(key)).encrypt(bytes(iv), bytes(data), None)
    return out[:-16], out[-16:]


def payload(data: bytes, mode: str) -> tuple[bytes, bool]:
    """(payload, compressed): `mode`'s zstd frame when it is smaller than the chunk, else the chunk."""
    data = bytes(data)
    frame = FRAMES[mode]
    if frame is not None and data:
        fr = frame(data)
        if len(fr) < len(data):
            return fr, True
    return data, False


def blob_encode_enc(key: bytes, iv: bytes, data: bytes, mode: str = "raw") -> bytes:
    pl, comp = payload(data, mode)
    ct, tag = gcm_encrypt(key, iv, pl)
    magic = ENCR_COMPR_BLOB_MAGIC_1_0 if comp else ENCRYPTED_BLOB_MAGIC_1_0
    return magic + zlib.crc32(ct).to_bytes(4, "little") + bytes(iv) + tag + ct


def blob_decrypt(key: bytes, blob: bytes) -> tuple[bytes, bool]:
    """(payload, compressed) of an encrypted blob; raises cryptography's InvalidTag when the tag does not verify and
    ValueError on a bad magic or CRC."""
    magic, crc, iv, tag, ct = blob[:8], blob[8:12], blob[12:28], blob[28:44], blob[44:]
    if magic not in MAGIC_LABELS:
        raise ValueError("not an encrypted blob")
    if int.from_bytes(crc, "little") != zlib.crc32(ct):
        raise ValueError("blob CRC mismatch")
    return AESGCM(bytes(key)).decrypt(bytes(iv), bytes(ct) + bytes(tag), None), magic == ENCR_COMPR_BLOB_MAGIC_1_0


# ---- GF(2^128) in Python integers, GCM bit order (bit 0 of the block = coefficient x^0 = the integer's top bit) -----
# Used to build test inputs (IVs with a chosen J0) and to restate GCM from the AES block function alone.
R = 0xE1 << 120
ONE = 1 << 127


def gf_mul(x: int, y: int) -> int:
    z, v = 0, y
    for i in range(127, -1, -1):
        if (x >> i) & 1:
            z ^= v
        v = (v >> 1) ^ (R if v & 1 else 0)
    return z


def gf_pow(h: int, k: int) -> int:
    r = ONE
    while k:
        if k & 1:
            r = gf_mul(r, h)
        h, k = gf_mul(h, h), k >> 1
    return r


def blocks(b: bytes) -> list[int]:
    b = bytes(b) + bytes(-len(b) % 16)
    return [int.from_bytes(b[i:i + 16], "big") for i in range(0, len(b), 16)]


def ghash(h: int, xs: list[int]) -> int:
    y = 0
    for x in xs:
        y = gf_mul(y ^ x, h)
    return y


def aes_block(key: bytes, x: int) -> int:
    e = Cipher(algorithms.AES(bytes(key)), modes.ECB()).encryptor()
    return int.from_bytes(e.update(x.to_bytes(16, "big")) + e.finalize(), "big")


def j0_of(key: bytes, iv: bytes) -> int:
    """J0 of a 16-byte IV: GHASH_H(IV || 0^64 || [128]_64)."""
    return ghash(aes_block(key, 0), blocks(iv) + [128])


def iv_for_j0(key: bytes, j0: int) -> bytes:
    """The 16-byte IV whose J0 is `j0`: J0 = (IV * H ^ 128) * H, solved with H^-1 = H^(2^128 - 2)."""
    hinv = gf_pow(aes_block(key, 0), (1 << 128) - 2)
    return (gf_mul(gf_mul(j0, hinv) ^ 128, hinv)).to_bytes(16, "big")
