"""The sparse file restore without a GPU: tests/file_sparse_ref.py's extents are the complement of the all-zero
file-aligned 4 KiB block parts, the ceil(B / 2) bound holds and is reached, a file read in block-aligned pieces gives
the whole file's extents, the zero-chunk rule picks exactly the longest all-zero chunks of a payload stream as the
chunker cuts it, and both file-sparse calls are exported, declared in plain C and bound in _lib's signature table."""
import ctypes as C
import hashlib
import random
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

import file_sparse_ref as fr
import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent
B = fr.BLOCK


def zero_run_file(size: int, seed: int) -> bytes:
    """Random bytes with zero runs starting and ending at every alignment around 4096, a zero head and a zero tail."""
    rng = random.Random(seed)
    a = bytearray(rng.randbytes(size))
    for lo in range(0, size, B):
        for d in (-3, -1, 0, 1, 15, 16):
            if rng.random() < 0.3:
                s = max(0, lo + d)
                n = rng.choice([1, 15, 16, B - 1, B, B + 1, 2 * B + d, 3 * B])
                a[s:s + n] = bytes(len(a[s:s + n]))
    a[:B + 5] = bytes(B + 5)
    a[size - 2 * B - 7:] = bytes(2 * B + 7)
    return bytes(a)


def check_complement(content: bytes, pos: int, length: int) -> list[tuple[int, int]]:
    ext = fr.extents(content, pos, length)
    assert all(a + n < b for (a, n), (b, _) in zip(ext, ext[1:])), "extents ascending and maximal"
    m = np.zeros(length, bool)
    for a, n in ext:
        assert pos <= a and a + n <= pos + length and n > 0
        m[a - pos:a - pos + n] = True
    v = np.frombuffer(content, np.uint8)
    lo = pos
    while lo < pos + length:   # block parts aligned to the content start
        hi = min(pos + length, (lo // B + 1) * B)
        part = m[lo - pos:hi - pos]
        assert part.all() or not part.any(), (lo, hi)
        assert bool(part[0]) == bool(v[lo:hi].any()), (lo, hi)
        lo = hi
    assert fr.packed(content, ext) == bytes(v[pos:pos + length][m])
    assert len(ext) <= fr.ext_bound(pos, length)
    return ext


@pytest.mark.parametrize("seed", range(3))
def test_extents_are_the_complement_of_the_zero_block_parts(seed):
    rng = random.Random(200 + seed)
    size = 19 * B + rng.randrange(B)
    f = zero_run_file(size, seed)
    ranges = [(0, size), (0, 0), (size, 0), (size - 1, 1), (B - 1, 2), (1, B), (B + 7, 3 * B - 9)]
    for _ in range(150):
        a = rng.randrange(0, size + 1)
        ranges.append((a, rng.randrange(0, size - a + 1)))
    for a, n in ranges:
        check_complement(f, a, n)


@pytest.mark.parametrize("piece", [B, 3 * B, 16 * B])
def test_block_aligned_pieces_give_the_whole_files_extents(piece):
    f = zero_run_file(21 * B + 1234, 7)
    whole = fr.extents(f, 0, len(f))
    merged: list[tuple[int, int]] = []
    for lo in range(0, len(f), piece):
        for a, n in check_complement(f, lo, min(piece, len(f) - lo)):
            if merged and merged[-1][0] + merged[-1][1] == a:
                merged[-1] = (merged[-1][0], merged[-1][1] + n)
            else:
                merged.append((a, n))
    assert merged == whole


@pytest.mark.parametrize("pos,length", [(0, 8 * B), (1, 7 * B + 5), (B - 1, 9 * B), (0, 1), (B - 1, 2), (0, 15 * B + 1)])
def test_the_extent_bound_is_reached_by_alternating_blocks(pos, length):
    f = b"".join((b"\x5a" * B if k % 2 == 0 else bytes(B)) for k in range(18))
    ext = check_complement(f, pos, length)
    assert len(ext) == fr.ext_bound(pos, length)


@pytest.mark.parametrize("seed", range(8))
def test_a_zero_window_hashes_to_zero_under_any_table(seed):
    t = np.random.default_rng(seed).integers(0, 1 << 32, 256, dtype=np.uint64).astype(np.uint32)
    assert fr.zero_window_hash(t) == 0
    assert len(fr.scan_ref.candidates(t, (1 << 12) - 1, bytes(5000))) == 0


@pytest.mark.parametrize("avg", [4 << 10, 64 << 10])
def test_the_zero_chunk_rule_picks_the_longest_all_zero_chunks(avg):
    """A payload stream of files with zero runs, cut as PayloadStreamWriter's chunker cuts it: the rule picks exactly
    the all-zero chunks of the longest length, and inside an all-zero file every zero chunk but the ones touching its
    ends has that length."""
    cfg = pg.make_config(avg)
    mx = int(cfg.max)
    rng = np.random.default_rng(avg)
    files = [bytes(3 * mx + 5), rng.integers(0, 256, 5000, dtype=np.uint8).tobytes() + bytes(4 * mx) + b"\x01",
             b"", b"\x07", zero_run_file(5 * mx // B * B + 99, 3), bytes(mx * 2 + 1)]
    stream, offs = fr.payload_stream(files)
    ends = fr.stream_ends(cfg, stream, offs)
    assert ends[-1] == len(stream)
    starts = [0] + ends[:-1]
    digs = [hashlib.sha256(stream[a:e]).digest() for a, e in zip(starts, ends)]
    lens = [e - a for a, e in zip(starts, ends)]
    assert max(lens) == mx
    want = {k for k, (a, e) in enumerate(zip(starts, ends)) if e - a == mx and stream[a:e].count(0) == mx}
    assert fr.zero_chunks(ends, digs) == want
    assert len(want) >= 5
    ident = bytes(range(32))
    keyed = [hashlib.sha256(stream[a:e] + ident).digest() for a, e in zip(starts, ends)]
    assert fr.zero_chunks(ends, keyed, ident) == want and fr.zero_chunks(ends, digs, ident) == set()
    # the first file is all zeros: between its first and last chunk every chunk is a zero chunk of the maximum
    lo, hi = offs[0] + 16, offs[0] + 16 + len(files[0])
    inner = [k for k, (a, e) in enumerate(zip(starts, ends)) if a >= lo and e <= hi]
    assert inner and set(inner) <= want and sum(lens[k] for k in inner) > len(files[0]) - 2 * mx


def test_a_longest_digest_held_once_serves_no_chunk_by_digest():
    """The zero digest is computed only when a digest of the longest length repeats: a lone longest zero chunk is read
    like a data chunk (its extents do not change), while two of them are both served by digest."""
    z = fr.sparse_ref.zero_digest(300)
    other = bytes(range(32))
    ends = [100, 400, 500, 800, 850]   # lengths 100, 300, 100, 300, 50
    assert fr.zero_chunks(ends, [other, z, other, other[::-1], other]) == set()
    assert fr.zero_chunks(ends, [other, z, other, z, other]) == {1, 3}
    assert fr.zero_chunks(ends, [other, other, z, other, z]) == set()   # a repeat, but not of zeros
    assert fr.zero_chunks([], []) == set()


def test_file_sparse_calls_are_exported_and_bound():
    L = _lib.lib()
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    for name, nargs, u32, u64 in (("pbsgpu_reader_plan_file_sparse", 10, [5], [8]),
                                  ("pbsgpu_reader_read_file_sparse", 18, [5, 10], [14])):
        assert hasattr(L, name)
        sig = _lib._SIGNATURES[name]
        assert len(sig) == nargs
        assert [k for k, t in enumerate(sig) if t is C.c_uint32] == u32
        assert [k for k, t in enumerate(sig) if t is C.c_uint64] == u64
        decl = re.search(rf"int {name}\(([^;]*)\);", hdr).group(1)
        params = [p.strip() for p in decl.split(",")]
        assert len(params) == nargs
        assert [k for k, p in enumerate(params) if p.startswith("uint32_t ")] == u32
        assert [k for k, p in enumerate(params) if p.startswith("uint64_t ") and "*" not in p] == u64


def test_file_sparse_declarations_are_plain_c(tmp_path):
    src = tmp_path / "f.c"
    src.write_text(r'''
#include "pbsgpu.h"
int main(void) {
    int (*p)(pbsgpu_reader *, const uint64_t *, const uint64_t *, const uint64_t *, const uint64_t *, uint32_t,
             uint64_t *, uint8_t *, uint64_t, uint64_t *) = pbsgpu_reader_plan_file_sparse;
    int (*r)(pbsgpu_reader *, const uint64_t *, const uint64_t *, const uint64_t *, const uint64_t *, uint32_t,
             const void *, const uint64_t *, const uint64_t *, const uint64_t *, uint32_t, uint8_t *, const uint64_t *,
             uint64_t *, uint64_t, uint64_t *, int32_t *, int32_t *) = pbsgpu_reader_read_file_sparse;
    uint64_t n;
    /* NULL reader: argument errors before any work, no device needed */
    return p(NULL, NULL, NULL, NULL, NULL, 0, NULL, NULL, 0, &n) == PBSGPU_EINVAL
        && r(NULL, NULL, NULL, NULL, NULL, 0, NULL, NULL, NULL, NULL, 0, NULL, NULL, NULL, 0, NULL, NULL, NULL) == PBSGPU_EINVAL
        ? 0 : 1;
}
''')
    exe = tmp_path / "f.bin"
    lib = ROOT / "pbs_plus_b200"
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-I", str(ROOT / "include"), "-o", str(exe), str(src),
                           f"-L{lib}", "-lpbsgpu", f"-Wl,-rpath,{lib}"])
    assert subprocess.run([str(exe)]).returncode == 0


def test_the_extent_writer_leaves_holes(tmp_path):
    """RestoreFiles' write side: one pwrite per extent into a new file, then ftruncate to the size, leaves every block
    outside the extents a hole (checked with SEEK_DATA; skipped where the filesystem does not report holes)."""
    import errno
    import os

    from pbs_plus_b200 import transfer
    f = zero_run_file(64 * B + 77, 11)
    ext = fr.extents(f, 0, len(f))
    p = tmp_path / "f"
    fd = os.open(p, os.O_CREAT | os.O_TRUNC | os.O_RDWR, 0o600)
    try:
        transfer._write_extents(fd, ext, fr.packed(f, ext))
        os.ftruncate(fd, len(f))
        assert os.pread(fd, len(f) + 1, 0) == f
        try:
            first = os.lseek(fd, 0, os.SEEK_DATA)
        except OSError:
            first = -1
        if first != ext[0][0]:
            pytest.skip("this filesystem does not report holes (SEEK_DATA)")
        at = 0
        for a, n in ext:   # data exactly where the extents are, a hole up to each of them
            assert os.lseek(fd, at, os.SEEK_DATA) == a
            assert os.lseek(fd, a, os.SEEK_HOLE) >= a + n
            at = a + n
        if at < len(f) // B * B:
            with pytest.raises(OSError) as e:
                os.lseek(fd, at if at % B == 0 else (at // B + 1) * B, os.SEEK_DATA)
            assert e.value.errno == errno.ENXIO
    finally:
        os.close(fd)
