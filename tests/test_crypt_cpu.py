"""CPU checks of encrypt mode: tests/crypt_ref.py against the GCM specification's vectors and against a GCM built here
from the AES block function alone (which also restates the segment / lane split of K11's GHASH), the two encrypted-blob
magics re-derived from their labels, and the C ABI's new entry points that need no GPU."""
import ctypes as C
import hashlib
import os
import random
import re
from pathlib import Path

import pytest
from cryptography.exceptions import InvalidTag

import crypt_ref
from pbs_plus_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent
LENGTHS = (0, 1, 15, 16, 17, 4095, (1 << 20) + 3)

gf_mul, gf_pow, blocks, ghash, aes_block = (crypt_ref.gf_mul, crypt_ref.gf_pow, crypt_ref.blocks, crypt_ref.ghash,
                                            crypt_ref.aes_block)


def ghash_split(h: int, xs: list[int], lanes: int, lane_blocks: int) -> int:
    """K11's order of the same sum: segments of lanes x lane_blocks blocks; lane l runs Horner with the step
    H^lanes over blocks l, l + lanes, ... and scales by H^(segment end - its last block); the segments are chained by
    Horner with H^(blocks of the segment); then (A * H ^ last) * H appends the last block (the length block)."""
    data, last = xs[:-1], xs[-1]
    w, hl = lanes * lane_blocks, gf_pow(h, lanes)
    a = 0
    for s0 in range(0, len(data), w):
        e = min(s0 + w, len(data)) - 1
        q = 0
        for lane in range(lanes):
            y, lb = 0, None
            for b in range(s0 + lane, e + 1, lanes):
                y, lb = gf_mul(y, hl) ^ data[b], b
            if lb is not None:
                q ^= gf_mul(y, gf_pow(h, e - lb))
        a = (gf_mul(a, gf_pow(h, e + 1 - s0)) if s0 else 0) ^ q
    return gf_mul(gf_mul(a, h) ^ last, h)


def gcm_from_block(key: bytes, iv: bytes, data: bytes, aad: bytes = b"", split=None) -> tuple[bytes, bytes]:
    h = aes_block(key, 0)
    if len(iv) == 12:
        j0 = int.from_bytes(iv + b"\0\0\0\1", "big")
    else:
        j0 = ghash(h, blocks(iv) + [len(iv) * 8])   # the general path (crypt_ref.j0_of for 16 bytes)
    ks = bytearray()
    for i in range((len(data) + 15) // 16):
        ctr = (j0 & ~0xFFFFFFFF) | ((j0 + i + 1) & 0xFFFFFFFF)      # inc32: the low word wraps
        ks += aes_block(key, ctr).to_bytes(16, "big")
    ct = bytes(a ^ b for a, b in zip(data, ks))
    lens = (len(aad) * 8) << 64 | len(ct) * 8
    if split:
        assert not aad
        s = ghash_split(h, blocks(ct) + [lens], *split)
    else:
        s = ghash(h, blocks(aad) + blocks(ct) + [lens])
    return ct, (s ^ aes_block(key, j0)).to_bytes(16, "big")


# ---- the GCM specification (McGrew / Viega), 256-bit key, IVs of 8 and 60 bytes (test cases 17 and 18) ---------------
K = bytes.fromhex("feffe9928665731c6d6a8f9467308308" * 2)
P = bytes.fromhex("d9313225f88406e5a55909c5aff5269a86a7a9531534f7da2e4c303d8a318a721c3c0c95956809532fcf0e2449a6b525"
                  "b16aedf5aa0de657ba637b39")
A = bytes.fromhex("feedfacedeadbeeffeedfacedeadbeefabaddad2")
SPEC = [
    (bytes.fromhex("cafebabefacedbad"),
     "c3762df1ca787d32ae47c13bf19844cbaf1ae14d0b976afac52ff7d79bba9de0feb582d33934a4f0954cc2363bc73f7862ac430e64abe499"
     "f47c9b1f", "3a337dbf46a792c45e454913fe2ea8f2"),
    (bytes.fromhex("9313225df88406e555909c5aff5269aa6a7a9538534f7da1e4c303d2a318a728c3c0c95156809539fcf0e2429a6b5254"
                   "16aedbf5a0de6a57a637b39b"),
     "5a8def2f0c9e53f1f75d7853659e2a20eeb2b22aafde6419a058ab4f6f746bf40fc0c3b780f244452da3ebf1c5d82cdea2418997200ef82e"
     "44ae7e3f", "a44a8266ee1c8eb0c8b5d4cf5ae9f19a"),
]


@pytest.mark.parametrize("iv,ct,tag", SPEC)
def test_gcm_spec_vectors_with_a_long_iv(iv, ct, tag):
    from cryptography.hazmat.primitives.ciphers.aead import AESGCM
    assert AESGCM(K).encrypt(iv, P, A) == bytes.fromhex(ct + tag)
    assert gcm_from_block(K, iv, P, A) == (bytes.fromhex(ct), bytes.fromhex(tag))


@pytest.mark.parametrize("n", LENGTHS)
def test_restatement_equals_gcm_from_the_block_function_with_16_byte_ivs(n):
    rng = random.Random(n)
    key, iv = rng.randbytes(32), rng.randbytes(16)
    data = rng.randbytes(n)
    ct, tag = crypt_ref.gcm_encrypt(key, iv, data)
    if n <= 4095:
        assert (ct, tag) == gcm_from_block(key, iv, data)
    else:   # the block-by-block model is slow in Python: check the head and the tag's algebra on a prefix
        head = data[:4096 + 5]
        assert crypt_ref.gcm_encrypt(key, iv, head) == gcm_from_block(key, iv, head)
        assert ct[:len(head)] == crypt_ref.gcm_encrypt(key, iv, head)[0]
    assert crypt_ref.gcm_encrypt(key, iv, data) == (ct, tag)


def test_inc32_wraps_inside_a_message():
    """An IV whose J0 low word is 0xFFFFFFF0: the 16th counter block wraps to low word 0 without a carry."""
    key = bytes(range(32))
    j0 = 0x0123456789ABCDEF_00112233_FFFFFFF0
    iv = crypt_ref.iv_for_j0(key, j0)
    assert crypt_ref.j0_of(key, iv) == j0
    data = os.urandom(16 * 40 + 7)
    assert crypt_ref.gcm_encrypt(key, iv, data) == gcm_from_block(key, iv, data)


@pytest.mark.parametrize("lanes,lane_blocks", [(32, 2), (4, 3), (1, 5)])
@pytest.mark.parametrize("n", (0, 1, 16, 17, 200, 1000, 1537))
def test_segment_and_lane_split_of_ghash_gives_the_tag(lanes, lane_blocks, n):
    rng = random.Random(n * 7 + lanes)
    key, iv, data = rng.randbytes(32), rng.randbytes(16), rng.randbytes(n)
    assert gcm_from_block(key, iv, data, split=(lanes, lane_blocks)) == crypt_ref.gcm_encrypt(key, iv, data)


def test_encrypted_blob_layout_and_tamper_detection():
    key, iv = bytes(range(32)), bytes(range(100, 116))
    data = b"hello " * 5000 + bytes(300_000)   # the zero run makes every mode, _z included, compress
    for mode in crypt_ref.FRAMES:
        blob = crypt_ref.blob_encode_enc(key, iv, data, mode)
        assert blob[12:28] == iv and len(blob) - crypt_ref.HEADER == len(crypt_ref.payload(data, mode)[0])
        pl, comp = crypt_ref.blob_decrypt(key, blob)
        assert comp == (mode != "raw") and pl == crypt_ref.payload(data, mode)[0]
        bad = bytearray(blob)
        bad[crypt_ref.HEADER + 3] ^= 0x10
        bad[8:12] = __import__("zlib").crc32(bytes(bad[44:])).to_bytes(4, "little")
        with pytest.raises(InvalidTag):
            crypt_ref.blob_decrypt(key, bytes(bad))


def test_id_key_and_keyed_digest():
    key = bytes(range(32))
    ident = crypt_ref.id_key(key)
    assert ident == hashlib.pbkdf2_hmac("sha256", key, b"_id_key", 10, 32) and len(ident) == 32
    assert crypt_ref.compute_digest(b"abc", ident) == hashlib.sha256(b"abc" + ident).digest()
    assert crypt_ref.compute_digest(b"abc", ident) != hashlib.sha256(b"abc").digest()


def test_encrypted_blob_magics_are_the_sha256_prefixes_upstream_derives_them_from():
    for magic, label in crypt_ref.MAGIC_LABELS.items():
        assert hashlib.sha256(label.encode()).digest()[:8] == magic, label


def test_product_never_imports_cryptography():
    for p in (ROOT / "pbs_plus_b200").rglob("*.py"):
        txt = p.read_text()
        assert not re.search(r"^\s*(import|from)\s+cryptography\b", txt, re.M), p


def test_crypt_entry_points_are_declared_exported_and_checked():
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    L = _lib.lib()
    for s in ("pbsgpu_crypt_create", "pbsgpu_crypt_destroy", "pbsgpu_blob_size_enc", "pbsgpu_blob_encode_batch_enc"):
        assert re.search(rf"\b{s}\s*\(", hdr) and s in _lib.SYMBOLS and hasattr(L, s), s
    assert [L.pbsgpu_blob_size_enc(n) for n in (0, 1, 1 << 24)] == [44, 45, (1 << 24) + 44]
    h = C.c_void_p()
    assert L.pbsgpu_crypt_create(None, bytes(32), C.byref(h)) == _lib.EINVAL and not h.value
    L.pbsgpu_crypt_destroy(None)
    assert L.pbsgpu_blob_encode_batch_enc(None, None, 1, None, None, None, 0, None, None, None, None, None) == _lib.EINVAL


def test_batch_opts_keeps_the_old_layout_in_front_of_crypt():
    """A caller built against the header without `crypt` passes size 48; the library accepts that size (GPU test)."""
    assert _lib.BatchOpts.crypt.offset == 48 and C.sizeof(_lib.BatchOpts) == 56


# tests/golden/k3_sass_sha256.json holds the SHA-256 of every K3 kernel's SASS (addresses stripped), plain and keyed, as
# the nvcc named there compiles csrc/sha256.cu: a change to the kernels' code shows up here.
def test_sha256_kernels_compile_to_the_golden_sass(tmp_path):
    import json
    import shutil
    import subprocess
    from pbs_plus_b200 import build
    golden = json.loads((ROOT / "tests" / "golden" / "k3_sass_sha256.json").read_text())
    if not Path(build.NVCC).exists() or not shutil.which("cuobjdump"):
        pytest.skip("no nvcc / cuobjdump")
    ver = subprocess.run([build.NVCC, "--version"], capture_output=True, text=True).stdout
    if golden["nvcc"] not in ver:
        pytest.skip(f"the golden SASS is from nvcc {golden['nvcc']}")
    obj = tmp_path / "sha256.o"
    subprocess.check_call([build.NVCC, *build.FLAGS, "-c", str(ROOT / "pbs_plus_b200" / "csrc" / "sha256.cu"), "-o", str(obj)])
    for name, want in golden["kernels"].items():
        txt = subprocess.run(["cuobjdump", "-sass", "-fun", name, str(obj)], capture_output=True, text=True).stdout
        lines = [re.sub(r"/\*[0-9a-f]{4,5}\*/", "", ln).strip() for ln in txt.splitlines()
                 if re.search(r"/\*[0-9a-f]{4,5}\*/|/\* 0x", ln)]
        assert lines and hashlib.sha256("\n".join(lines).encode()).hexdigest() == want, name
