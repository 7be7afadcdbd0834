"""The sparse image restore without a GPU: tests/sparse_ref.py's extents are exactly the complement of the all-zero
image-aligned 4 KiB block parts, the ceil(B / 2) extent bound holds and is reached, and pbsgpu_reader_read_sparse is
exported, declared in plain C and bound in _lib's signature table."""
import ctypes as C
import hashlib
import random
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import sparse_ref
from pbs_plus_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent
B = sparse_ref.BLOCK


def zero_run_image(size: int, seed: int) -> bytes:
    """Random bytes with zero runs that start and end at every alignment around 4096 (and at random places)."""
    rng = random.Random(seed)
    a = bytearray(rng.randbytes(size))
    for lo in range(0, size, B):
        for d in (-3, -1, 0, 1, 15, 16):
            if rng.random() < 0.3:
                s = max(0, lo + d)
                n = rng.choice([1, 15, 16, B - 1, B, B + 1, 2 * B + d, 3 * B])
                a[s:s + n] = bytes(len(a[s:s + n]))
    return bytes(a)


def covered(ext, off, length) -> np.ndarray:
    """Per byte of the range: inside one of its extents."""
    m = np.zeros(length, bool)
    for a, n in ext:
        assert off <= a and a + n <= off + length and n > 0
        m[a - off:a - off + n] = True
    return m


def check_complement(img: bytes, off: int, length: int) -> None:
    ext = sparse_ref.extents(img, off, length)
    assert all(a + n < b for (a, n), (b, _) in zip(ext, ext[1:])), "extents ascending and maximal"
    m = covered(ext, off, length)
    v = np.frombuffer(img, np.uint8)
    # block by block, image-aligned: a part is outside every extent exactly when all its bytes are zero
    lo = off
    while lo < off + length:
        hi = min(off + length, (lo // B + 1) * B)
        part = m[lo - off:hi - off]
        assert part.all() or not part.any(), (lo, hi)
        assert bool(part[0]) == bool(v[lo:hi].any()), (lo, hi)
        lo = hi
    assert sparse_ref.packed(img, ext) == bytes(v[off:off + length][m])
    assert len(ext) <= sparse_ref.ext_bound(off, length)


@pytest.mark.parametrize("seed", range(4))
def test_extents_are_the_complement_of_the_zero_block_parts(seed):
    rng = random.Random(100 + seed)
    size = 23 * B + rng.randrange(B)
    img = zero_run_image(size, seed)
    ranges = [(0, size), (0, 0), (size, 0), (B, 0), (size - 1, 1), (0, 1), (B - 1, 1), (B, 1), (B - 1, 2), (1, B),
              (B + 7, 3 * B - 9)]
    for _ in range(200):
        a = rng.randrange(0, size + 1)
        ranges.append((a, rng.randrange(0, size - a + 1)))
    for a, n in ranges:
        check_complement(img, a, n)
        if n == 0:
            assert sparse_ref.extents(img, a, n) == [] and sparse_ref.ext_bound(a, n) == 0


def test_single_byte_ranges_follow_their_byte():
    img = bytes([0, 1] * (B // 2)) + bytes(B) + b"\x07"
    for a in range(0, len(img), 97):
        assert sparse_ref.extents(img, a, 1) == ([(a, 1)] if img[a] else [])


def test_block_parts_are_image_aligned():
    assert sparse_ref.block_parts(B - 1, B + 2) == [(B - 1, B), (B, 2 * B), (2 * B, 2 * B + 1)]
    assert sparse_ref.block_parts(5, 10) == [(5, 15)]
    assert sparse_ref.block_parts(3 * B, 0) == []


@pytest.mark.parametrize("start,length", [(0, 8 * B), (1, 7 * B + 5), (B - 1, 9 * B), (100, 1), (0, 1), (B - 1, 2),
                                          (5, 2 * B), (0, 15 * B + 1)])
def test_the_extent_bound_is_reached_by_alternating_blocks(start, length):
    """Even blocks data, odd blocks zero, a range starting in block 2: its parts alternate data and hole from a data
    part on, so it has ceil(B / 2) extents, one per data part."""
    img = b"".join((b"\x5a" * B if k % 2 == 0 else bytes(B)) for k in range(20))
    off = 2 * B + start
    ext = sparse_ref.extents(img, off, length)
    assert len(ext) == sparse_ref.ext_bound(off, length) == (len(sparse_ref.block_parts(off, length)) + 1) // 2
    check_complement(img, off, length)


def test_zero_digests_plain_and_keyed():
    assert sparse_ref.zero_digest(4096) == hashlib.sha256(bytes(4096)).digest()
    ident = bytes(range(32))
    assert sparse_ref.zero_digest(10, ident) == hashlib.sha256(bytes(10) + ident).digest()


def test_read_sparse_is_exported_and_bound():
    L = _lib.lib()
    assert hasattr(L, "pbsgpu_reader_read_sparse")
    sig = _lib._SIGNATURES["pbsgpu_reader_read_sparse"]
    assert len(sig) == 17 and sig[3] == C.c_uint32 and sig[9] == C.c_uint32 and sig[13] == C.c_uint64
    assert _lib.READ_SPARSE == 4 and _lib.SPARSE_BLOCK == B
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    assert re.search(r"#define PBSGPU_READ_SPARSE 4u", hdr)
    decl = re.search(r"int pbsgpu_reader_read_sparse\(([^;]*)\);", hdr).group(1)
    assert decl.count(",") == 16


def test_read_sparse_declaration_is_plain_c(tmp_path):
    src = tmp_path / "s.c"
    src.write_text(r'''
#include "pbsgpu.h"
int main(void) {
    int (*f)(pbsgpu_reader *, const uint64_t *, const uint64_t *, uint32_t, uint32_t, const void *, const uint64_t *,
             const uint64_t *, const uint64_t *, uint32_t, uint8_t *, const uint64_t *, uint64_t *, uint64_t, uint64_t *,
             int32_t *, int32_t *) = pbsgpu_reader_read_sparse;
    /* NULL reader: argument error before any work, no device needed */
    return f(NULL, NULL, NULL, 0, 0, NULL, NULL, NULL, NULL, 0, NULL, NULL, NULL, 0, NULL, NULL, NULL) == PBSGPU_EINVAL
        && PBSGPU_READ_SPARSE == 4u ? 0 : 1;
}
''')
    exe = tmp_path / "s.bin"
    lib = ROOT / "pbs_plus_b200"
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-I", str(ROOT / "include"), "-o", str(exe), str(src),
                           f"-L{lib}", "-lpbsgpu", f"-Wl,-rpath,{lib}"])
    assert subprocess.run([str(exe)]).returncode == 0
