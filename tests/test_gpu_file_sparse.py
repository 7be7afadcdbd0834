"""The sparse file restore on the GPU (pbsgpu_reader_plan_file_sparse / _read_file_sparse, K17 + K14;
PayloadReader.RestoreFiles): payload archives written by PayloadStreamWriter at 4 KiB and 64 KiB averages, plain and
keyed, with all-zero files longer than the longest chunk, zero runs at unaligned offsets, zero heads and tails, zeros
across chunk boundaries, and empty and 1-byte files.  Extents and packed bytes equal tests/file_sparse_ref.py for whole
files and for pieces at aligned and unaligned offsets; zero chunks are never planned and need no blob; a wrong header
is BAD_HEADER only at pos 0; a corrupt blob fails only its ranges and leaves their output untouched; argument errors
leave the reader usable; the restore into a directory writes the bytes, keeps the holes, applies mode and mtime,
restores symlinks and skips a file that is already there."""
import errno
import io
import os
import random
import shutil
import stat
import tempfile
from pathlib import Path

import numpy as np
import pytest

import crypt_ref
import file_sparse_ref as fr
import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib, transfer
from pbs_plus_b200.engine import _blob_args, _ptr

pytestmark = pytest.mark.gpu
KEY = bytes(range(3, 35))
B = fr.BLOCK


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module", autouse=True)
def release_device_memory(torch):
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


def make_files(mx: int, seed: int) -> list[bytes]:
    rng = np.random.default_rng(seed)

    def rnd(n):
        return rng.integers(1, 256, n, dtype=np.uint8).tobytes()

    def holes(n):   # zero runs at unaligned offsets and across block bounds
        a = bytearray(rnd(n))
        for lo in range(0, n, 3 * B):
            s, k = lo + int(rng.integers(0, B)), int(rng.integers(1, 2 * B + 7))
            a[s:s + k] = bytes(len(a[s:s + k]))
        return bytes(a)

    return [
        bytes(3 * mx + 5),                                       # all zeros, longer than the longest chunk
        rnd(777) + bytes(4 * mx + 123) + rnd(5000),              # zeros across chunk boundaries, unaligned
        b"",
        b"\x07",
        bytes(B + 17) + rnd(3 * B) + bytes(2 * B + 3),           # zero head and tail
        holes(6 * B + 999),
        bytes(2 * mx) + b"\x01",                                 # a long zero head, one data byte at the end
        rnd(mx + 3),
        bytes(5),
    ]


def write_archive(eng, files: list[bytes], avg: int, key: bytes | None):
    """-> (didx, payload offsets, {digest: blob}, stream ends)"""
    store = {}
    w = transfer.PayloadStreamWriter(eng, pg.make_config(avg), upload_blob=lambda d, b: store.setdefault(d, b),
                                     blob_compression="lzh", crypt_key=key)
    offs = [w.WriteEntryReader(transfer.Entry(f"f{i}", len(f)), io.BytesIO(f), len(f)) for i, f in enumerate(files)]
    w.Finish()
    didx = w.didx()
    ends, _ = eng.didx_parse(didx)
    return didx, offs, store, [int(e) for e in ends]


def touched(ends, lo: int, hi: int) -> set[int]:
    """The chunks of the archive bytes [lo, hi); an empty span touches none."""
    if lo >= hi:
        return set()
    starts = [0] + ends[:-1]
    return {k for k, (a, e) in enumerate(zip(starts, ends)) if a < hi and e > lo and e > a}


def span(fo: int, pos: int, n: int) -> tuple[int, int]:
    """The archive bytes a range reads: its content, and its file's header at pos 0."""
    return (fo if pos == 0 else fo + 16 + pos), fo + 16 + pos + n


CASES = [(4 << 10, None), (64 << 10, None), (4 << 10, KEY), (64 << 10, KEY)]


@pytest.fixture(scope="module", params=CASES, ids=[f"{a >> 10}k-{'key' if k else 'plain'}" for a, k in CASES])
def archive(request, eng):
    avg, key = request.param
    mx = int(pg.make_config(avg).max)
    files = make_files(mx, avg + (1 if key else 0))
    didx, offs, store, ends = write_archive(eng, files, avg, key)
    _, dig = eng.didx_parse(didx)
    zeros = fr.zero_chunks(ends, dig, crypt_ref.id_key(key) if key else None)
    return dict(files=files, didx=didx, offs=offs, store=store, ends=ends, key=key, zeros=zeros, dig=dig, mx=mx, avg=avg)


def test_the_archive_is_cut_as_restated(archive):
    """The stream, its cuts and its zero chunks are the restatement's: every all-zero chunk of the longest length, and
    nothing else, is a zero chunk."""
    a = archive
    stream, offs = fr.payload_stream(a["files"])
    assert a["offs"] == offs and a["ends"] == fr.stream_ends(pg.make_config(a["avg"]), stream, offs)
    starts = [0] + a["ends"][:-1]
    assert a["zeros"] == {k for k, (s, e) in enumerate(zip(starts, a["ends"]))
                          if e - s == a["mx"] and stream[s:e].count(0) == e - s}
    assert len(a["zeros"]) >= 4


def open_reader(eng, a, cache_bytes=0):
    crypt = eng.crypt(a["key"]) if a["key"] else None
    return eng.reader(a["didx"], crypt, cache_bytes), crypt


def read(r, a, ranges, store=None):
    """ranges: (file index, pos, len) -> plan, fetch, read_file_sparse -> (chunks planned, status, data, bst)"""
    fo = [a["offs"][f] for f, _, _ in ranges]
    fs = [len(a["files"][f]) for f, _, _ in ranges]
    pos = [p for _, p, _ in ranges]
    ln = [n for _, _, n in ranges]
    chunks, dig = r.plan_file_sparse(fo, fs, pos, ln)
    st = a["store"] if store is None else store
    status, data, bst = r.read_file_sparse(fo, fs, pos, ln, {int(c): st[bytes(d)] for c, d in zip(chunks, dig)})
    return chunks.tolist(), status, data, bst


def check(a, ranges, status, data):
    assert status.tolist() == [0] * len(ranges)
    for (f, p, n), got in zip(ranges, data):
        c = a["files"][f]
        ext = fr.extents(c, p, n)
        assert got == (ext, fr.packed(c, ext)), (f, p, n)


def test_whole_files_and_pieces_equal_the_restatement(eng, archive):
    a = archive
    whole = [(f, 0, len(c)) for f, c in enumerate(a["files"])]
    rng = random.Random(len(a["ends"]))
    pieces = []
    for f, c in enumerate(a["files"]):
        n = len(c)
        for p in (B, 3 * B, 1, B - 1, 4097, n // 2, n - 1, n):
            if 0 < p <= n:
                pieces.append((f, p, rng.randrange(0, n - p + 1)))
        if n:
            pieces.append((f, 0, rng.randrange(0, n + 1)))
    r, crypt = open_reader(eng, a, cache_bytes=8 * a["mx"])
    try:
        for ranges in (whole, pieces, whole + pieces):
            r2, crypt2 = open_reader(eng, a)   # a cold cache: the plan names every data chunk
            try:
                chunks, st, data, bst = read(r2, a, ranges)
                want = set().union(*(touched(a["ends"], *span(a["offs"][f], p, n)) for f, p, n in ranges))
                assert chunks == sorted(want - a["zeros"])
                assert (bst == 0).all()
                check(a, ranges, st, data)
            finally:
                r2.close()
                if crypt2 is not None:
                    crypt2.close()
        # range by range through a small cache, and with every zero chunk's blob withheld
        no_zero = {d: b for d, b in a["store"].items() if d not in {bytes(a["dig"][k]) for k in a["zeros"]}}
        for rg in whole + pieces[::3]:
            chunks, st, data, _ = read(r, a, [rg], no_zero)
            assert not set(chunks) & a["zeros"]
            check(a, [rg], st, data)
    finally:
        r.close()
        if crypt is not None:
            crypt.close()


def raw_read(r, fo, fs, pos, ln, blobs, out, ext_cap=None):
    """pbsgpu_reader_read_file_sparse through ctypes with a caller-filled out -> (rc, status, ext, first, bst, oo)."""
    fo, fs, p, l = (np.array(x, np.uint64) for x in (fo, fs, pos, ln))
    base, bo, bl, bc = _blob_args(blobs)
    n, k = len(fo), len(bo)
    oo = np.zeros(n, np.uint64)
    oo[1:] = np.cumsum(l)[:-1]
    bound = sum(fr.ext_bound(int(x), int(y)) for x, y in zip(p, l))
    cap = bound if ext_cap is None else ext_cap
    ext = np.full((cap + 4, 2), 0xEEEE, np.uint64)
    first = np.zeros(n + 1, np.uint64)
    st, bst = np.zeros(n, np.int32), np.zeros(k, np.int32)
    rc = r._eng._L.pbsgpu_reader_read_file_sparse(
        r._h, fo.ctypes.data, fs.ctypes.data, p.ctypes.data, l.ctypes.data, n, _ptr(base), bo.ctypes.data,
        bl.ctypes.data, bc.ctypes.data, k, _ptr(out), oo.ctypes.data, ext.ctypes.data, cap, first.ctypes.data,
        st.ctypes.data, bst.ctypes.data)
    assert (ext[cap:] == 0xEEEE).all(), "extents written past ext_cap"
    return rc, st, ext[:cap], first, bst, oo


def test_wrong_header_only_at_pos_0(eng, archive):
    a = archive
    f = 1
    c = a["files"][f]
    fo, n = a["offs"][f], len(c)
    r, crypt = open_reader(eng, a)
    try:
        ranges = [(0, n - 1), (5, n - 6), (B, n - 1 - B)]   # the file as one byte shorter than its header says
        chunks, dig = r.plan_file_sparse([fo] * 3, [n - 1] * 3, [p for p, _ in ranges], [m for _, m in ranges])
        st, data, _ = r.read_file_sparse([fo] * 3, [n - 1] * 3, [p for p, _ in ranges], [m for _, m in ranges],
                                         {int(k): a["store"][bytes(d)] for k, d in zip(chunks, dig)})
        assert st.tolist() == [_lib.DEC_BAD_HEADER, 0, 0] and data[0] is None
        for (p, m), got in zip(ranges[1:], data[1:]):
            ext = fr.extents(c, p, m)
            assert got == (ext, fr.packed(c, ext))
    finally:
        r.close()
        if crypt is not None:
            crypt.close()


def test_corrupt_blob_fails_only_its_ranges(eng, archive):
    a = archive
    f = 1   # random head, a long zero run, a random tail: the head's chunk is a data chunk
    fo, c = a["offs"][f], a["files"][f]
    head = min(touched(a["ends"], fo + 16, fo + 17))
    assert head not in a["zeros"]
    blobs = {k: a["store"][bytes(a["dig"][k])] for k in range(len(a["ends"])) if k not in a["zeros"]}
    bad = bytearray(blobs[head]); bad[-1] ^= 0x40; blobs[head] = bytes(bad)
    tail = len(c) - 5000
    ranges = [(f, 0, len(c)), (f, tail, 5000), (7, 0, len(a["files"][7])), (f, 1, 100), (2, 0, 0)]
    fo_, fs_ = [a["offs"][g] for g, _, _ in ranges], [len(a["files"][g]) for g, _, _ in ranges]
    pos, ln = [p for _, p, _ in ranges], [n for _, _, n in ranges]
    r, crypt = open_reader(eng, a)
    try:
        out = np.full(sum(ln), 0xA5, np.uint8)
        rc, st, ext, first, bst, oo = raw_read(r, fo_, fs_, pos, ln, blobs, out)
        assert rc == 0
        want_bad = _lib.DEC_BAD_CRC   # the CRC comes before the GCM tag
        assert st.tolist() == [want_bad, 0, 0, want_bad, 0]
        assert [int(x) for x in bst] == [want_bad if k == head else 0 for k in blobs]
        for i, (g, p, n) in enumerate(ranges):
            e = [(int(x), int(y)) for x, y in ext[int(first[i]):int(first[i + 1])]]
            region = out[int(oo[i]):int(oo[i]) + n]
            if st[i]:
                assert e == [] and (region == 0xA5).all()
            else:
                want = fr.extents(a["files"][g], p, n)
                pk = fr.packed(a["files"][g], want)
                assert e == want and region[:len(pk)].tobytes() == pk and (region[len(pk):] == 0xA5).all()
    finally:
        r.close()
        if crypt is not None:
            crypt.close()


def test_argument_errors_leave_the_reader_usable(eng, archive):
    a = archive
    f = 5
    fo, c = a["offs"][f], a["files"][f]
    n = len(c)
    out = np.zeros(n + 16, np.uint8)
    size = a["ends"][-1]
    r, crypt = open_reader(eng, a)
    try:
        pos, ln = [1, B - 1, 0], [B - 1, 2 * B + 2, n]
        bound = sum(fr.ext_bound(p, m) for p, m in zip(pos, ln))
        assert raw_read(r, [fo] * 3, [n] * 3, pos, ln, {}, out, ext_cap=bound - 1)[0] == _lib.EINVAL
        assert raw_read(r, [fo], [n], [1], [n], {}, out)[0] == _lib.EINVAL            # past the file's end
        assert raw_read(r, [fo], [n], [n + 1], [0], {}, out)[0] == _lib.EINVAL
        assert raw_read(r, [size - 15], [0], [0], [0], {}, out)[0] == _lib.EINVAL      # header past the archive
        assert raw_read(r, [fo], [size], [0], [1], {}, out)[0] == _lib.EINVAL          # file past the archive
        for bad in (([fo], [n], [1], [n]), ([size], [0], [0], [0])):
            with pytest.raises(pg.PbsGpuError) as e:
                r.plan_file_sparse(*bad)
            assert e.value.code == _lib.EINVAL
        # the image form still refuses a .didx reader
        with pytest.raises(pg.PbsGpuError) as e:
            r.plan([0], [10], sparse=True)
        assert e.value.code == _lib.EINVAL
        with pytest.raises(pg.PbsGpuError) as e:
            r.read_sparse([0], [10], {})
        assert e.value.code == _lib.EINVAL
        # still usable
        chunks, st, data, _ = read(r, a, list(zip([f] * 3, pos, ln)))
        check(a, list(zip([f] * 3, pos, ln)), st, data)
    finally:
        r.close()
        if crypt is not None:
            crypt.close()


def test_an_image_reader_refuses_the_file_form(eng):
    data = bytes(8192) + os.urandom(4096)
    w = transfer.FixedIndexWriter(eng, 4096, eng.digest_set(), upload_blob=lambda d, b: None, blob_compression="z")
    w.WriteSlice(data)
    with eng.reader_fidx(w.fidx()) as r:
        with pytest.raises(pg.PbsGpuError) as e:
            r.plan_file_sparse([0], [10], [0], [10])
        assert e.value.code == _lib.EINVAL
        out = np.zeros(16, np.uint8)
        assert raw_read(r, [0], [10], [0], [10], {}, out)[0] == _lib.EINVAL


def seek_hole_works(tmp_path) -> bool:
    p = tmp_path / "probe"
    with open(p, "wb") as f:
        f.truncate(1 << 20)
        f.seek(512 << 10)
        f.write(b"x" * 4096)
    fd = os.open(p, os.O_RDONLY)
    try:
        return os.lseek(fd, 0, os.SEEK_DATA) > 0
    except OSError:
        return False
    finally:
        os.close(fd)


def whole_zero_blocks(c: bytes) -> list[tuple[int, int]]:
    out = []
    for lo in range(0, len(c) // B * B, B):
        if c[lo:lo + B].count(0) == B:
            if out and out[-1][1] == lo:
                out[-1] = (out[-1][0], lo + B)
            else:
                out.append((lo, lo + B))
    return out


@pytest.fixture
def hole_dir(tmp_path):
    """A directory on a filesystem that reports holes (SEEK_DATA): the test's own, else tmpfs at /dev/shm; skip when
    neither does, so the run records that holes were not checked."""
    if seek_hole_works(tmp_path):
        yield tmp_path
        return
    if os.path.isdir("/dev/shm"):
        d = Path(tempfile.mkdtemp(prefix="file_sparse_", dir="/dev/shm"))
        try:
            if seek_hole_works(d):
                yield d
                return
        finally:
            shutil.rmtree(d, ignore_errors=True)
    pytest.skip("no filesystem here reports holes (SEEK_DATA): holes not checked")


@pytest.mark.parametrize("slice_bytes", [1 << 30, 3 * B])
def test_restored_files_keep_their_holes(eng, archive, hole_dir, slice_bytes):
    """Every whole all-zero block of a restored file is a hole, and the all-zero file allocates next to nothing."""
    a = archive
    root = hole_dir / "r"
    entries = [transfer.FileEntry(f"f{i}", 0o100644, 0, o, len(c)) for i, (c, o) in enumerate(zip(a["files"], a["offs"]))]
    with transfer.PayloadReader(eng, a["didx"], a["store"].__getitem__, crypt_key=a["key"]) as pr:
        pr.RestoreFiles(str(root), entries, no_attr=True, slice_bytes=slice_bytes)
    checked = 0
    for e, c in zip(entries, a["files"]):
        p = root / e.path
        assert p.read_bytes() == c, e.path
        fd = os.open(p, os.O_RDONLY)
        try:
            for lo, hi in whole_zero_blocks(c):
                checked += 1
                try:
                    assert os.lseek(fd, lo, os.SEEK_DATA) >= hi, (e.path, lo, hi)
                except OSError as err:
                    assert err.errno == errno.ENXIO   # no data after lo: a hole to the end
        finally:
            os.close(fd)
    assert checked >= 10
    assert os.stat(root / "f0").st_blocks * 512 < len(a["files"][0]) // 8


@pytest.mark.parametrize("slice_bytes", [1 << 30, 3 * B])
def test_restore_files_into_a_directory(eng, archive, tmp_path, slice_bytes):
    a = archive
    zero_digs = {bytes(a["dig"][k]) for k in a["zeros"]}
    asked = []

    def source(d: bytes) -> bytes:
        asked.append(d)
        return a["store"][d]

    root = tmp_path / "r"
    entries = [transfer.DirEntry("d", 0o40750, 1_600_000_000), transfer.DirEntry("d/e", 0o40700, 1_600_000_100)]
    for i, (c, o) in enumerate(zip(a["files"], a["offs"])):
        entries.append(transfer.FileEntry(f"d/f{i}" if i % 2 else f"d/e/f{i}", 0o100640 | (i & 1) << 6,
                                          1_500_000_000 + i, o, len(c)))
    entries += [transfer.SymlinkEntry("d/link", "e/f0"), transfer.SymlinkEntry("top", "d")]
    files = {e.path: e for e in entries if isinstance(e, transfer.FileEntry)}
    with transfer.PayloadReader(eng, a["didx"], source, crypt_key=a["key"]) as pr:
        pr.RestoreFiles(str(root), entries, slice_bytes=slice_bytes)
        assert asked and not zero_digs & set(asked)
        for i, c in enumerate(a["files"]):
            e = files[f"d/f{i}" if i % 2 else f"d/e/f{i}"]
            p = root / e.path
            assert p.read_bytes() == c, e.path
            st = os.lstat(p)
            assert stat.S_IMODE(st.st_mode) == e.mode & 0o777 and int(st.st_mtime) == e.mtime
        assert os.readlink(root / "d/link") == "e/f0" and os.readlink(root / "top") == "d"
        for d in entries[:2]:
            st = os.stat(root / d.path)
            assert stat.S_IMODE(st.st_mode) == d.mode & 0o777 and int(st.st_mtime) == d.mtime
        # the skip rule: a file whose size and mtime match is not rewritten; one whose mtime differs is
        keep, redo = root / "d/f1", root / "d/e/f4"
        keep.write_bytes(b"\xee" * len(a["files"][1]))
        os.utime(keep, (files["d/f1"].mtime,) * 2)
        redo.write_bytes(b"\xee" * len(a["files"][4]))
        os.utime(redo, (1,) * 2)
        asked.clear()
        pr.RestoreFiles(str(root), entries, slice_bytes=slice_bytes)
        assert keep.read_bytes() == b"\xee" * len(a["files"][1])
        assert redo.read_bytes() == a["files"][4]
        assert stat.S_IMODE(os.stat(keep).st_mode) == files["d/f1"].mode & 0o777
        # no_attr: the mtime no longer matters, so the kept file stays even after its mtime moved
        os.utime(keep, (2,) * 2)
        pr.RestoreFiles(str(root), entries, no_attr=True, slice_bytes=slice_bytes)
        assert keep.read_bytes() == b"\xee" * len(a["files"][1]) and int(os.stat(keep).st_mtime) == 2


def test_restore_files_names_the_file_that_fails(eng, archive, tmp_path):
    a = archive
    f = 1
    fo = a["offs"][f]
    head = min(touched(a["ends"], fo + 16, fo + 17))
    store = dict(a["store"])
    d = bytes(a["dig"][head])
    store[d] = store[d][:-1] + bytes([store[d][-1] ^ 1])
    e = transfer.FileEntry("broken", 0o100644, 0, fo, len(a["files"][f]))
    with transfer.PayloadReader(eng, a["didx"], store.__getitem__, crypt_key=a["key"]) as pr:
        with pytest.raises(IOError, match=f"broken \\(payload offset {fo}"):
            pr.RestoreFiles(str(tmp_path / "x"), [e])
        with pytest.raises(ValueError):
            pr.RestoreFiles(str(tmp_path / "x"), [transfer.SymlinkEntry("../out", "x")])


@pytest.mark.parametrize("n_zero", [1, 2])
def test_a_lone_longest_zero_chunk_is_read_like_data(eng, n_zero):
    """An index cut by hand so that its longest chunks are all-zero ones: with one such chunk its digest is held once
    and the chunk is planned and read like a data chunk; with two, neither is planned.  The extents are the same."""
    L = 5 * B + 123
    rng = np.random.default_rng(n_zero)
    content = rng.integers(1, 256, 1000, dtype=np.uint8).tobytes() + bytes(L * n_zero) + \
        rng.integers(1, 256, 3000, dtype=np.uint8).tobytes()
    stream, (fo,) = fr.payload_stream([content])
    e0 = fo + 16 + 1000
    ends = [e0] + [e0 + L * (k + 1) for k in range(n_zero)] + [len(stream)]
    a = np.frombuffer(stream, np.uint8)
    off = np.array([0] + ends[:-1], np.uint64)
    ln = np.array(ends, np.uint64) - off
    dig = eng.sha256_batch(a, off, ln)
    blobs = eng.blob_encode_batch_lzh(a, off, ln)[0]
    rec = np.zeros(len(ends), dtype=_lib.CHUNK_DTYPE)
    rec["end_off"] = ends
    rec["digest"] = dig
    with eng.reader(eng.didx_build(rec)) as r:
        chunks, _ = r.plan_file_sparse([fo], [len(content)], [0], [len(content)])
        zero = set(range(1, 1 + n_zero))
        assert fr.zero_chunks(ends, dig) == (zero if n_zero > 1 else set())
        assert chunks.tolist() == sorted(set(range(len(ends))) - fr.zero_chunks(ends, dig))
        st, data, _ = r.read_file_sparse([fo], [len(content)], [0], [len(content)],
                                         {int(c): blobs[int(c)] for c in chunks})
        ext = fr.extents(content, 0, len(content))
        assert st.tolist() == [0] and data[0] == (ext, fr.packed(content, ext))
