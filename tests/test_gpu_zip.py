"""The zip restore on the GPU: pbsgpu_reader_read_deflate on _z and _lzh payload archives, plain and encrypted (each
stream inflates to ReadFileContents' bytes); a corrupt blob sets only its own ranges' status, with out_len 0 and the
sentinel bytes of those ranges untouched; a call that decodes in groups; and transfer.ZipWriter end to end -- a tree
with empty files and directories, symlinks, non-ASCII names and a 1 GiB file extracted by zipfile equal to the source
with its modes and mtimes, and one file of 4 GiB + 1 zeros written in pieces with zip64 sizes."""
import io
import os
import stat
import zipfile
import zlib

import numpy as np
import pytest

import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib, engine as E, transfer
from test_gpu_reader import KEY, SENT, content, file_sizes, write_snapshot

pytestmark = pytest.mark.gpu
AVG = 1 << 16


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


def inflate(s: bytes) -> bytes:
    return zlib.decompress(s, -15)


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "encrypted"])
@pytest.mark.parametrize("mode", ["z", "lzh"])
def test_read_deflate_inflates_to_the_files(eng, mode, key):
    files = [content(n, 700 + i) for i, n in enumerate(file_sizes(pg.make_config(AVG)))]
    didx, offs, archive, store = write_snapshot(eng, files, mode, key)
    with transfer.PayloadReader(eng, didx, store.__getitem__, crypt_key=key) as r:
        want = r.ReadFileContents(list(zip(offs, [len(f) for f in files])))
        streams, crcs = r._read_deflate(offs, [len(f) for f in files], True)
        assert [inflate(s) for s in streams] == want == files
        assert crcs == [zlib.crc32(f) for f in files]
        # plain ranges across chunk edges
        ends = [int(x) for x in eng.didx_parse(didx)[0]]
        rng = [(ends[1] - 9, ends[4] - ends[1] + 20), (3, 1000), (ends[2], 0)]
        streams, _ = r._read_deflate([o for o, _ in rng], [n for _, n in rng], False)
        assert [inflate(s) for s in streams] == [archive[o:o + n] for o, n in rng]


def raw_read_deflate(eng, r, off, ln, blobs, out, out_off, flags=0):
    o, l, oo = np.array(off, np.uint64), np.array(ln, np.uint64), np.array(out_off, np.uint64)
    items = list(blobs.items())
    bc = np.array([c for c, _ in items], np.uint64)
    bl = np.array([len(b) for _, b in items], np.uint64)
    bo = np.concatenate([[0], np.cumsum(bl)[:-1]]).astype(np.uint64) if items else np.zeros(0, np.uint64)
    base = np.frombuffer(b"".join(b for _, b in items) or b"\0", np.uint8)
    st = np.full(len(o), -1, np.int32)
    olen = np.full(len(o), 12345, np.uint64)
    crc = np.zeros(len(o), np.uint32)
    bst = np.full(len(items), -1, np.int32)
    eng._ck(eng._L.pbsgpu_reader_read_deflate(r._h, o.ctypes.data, l.ctypes.data, len(o), flags, None, base.ctypes.data,
                                              bo.ctypes.data, bl.ctypes.data, bc.ctypes.data, len(items), out.ctypes.data,
                                              oo.ctypes.data, olen.ctypes.data, crc.ctypes.data, st.ctypes.data,
                                              bst.ctypes.data))
    return st, olen, crc, bst


def test_a_corrupt_blob_fails_only_its_ranges(eng):
    files = [content(n, 800 + i) for i, n in enumerate([200_000, 300_000, 150_000])]
    didx, offs, archive, store = write_snapshot(eng, files, "lzh")
    ends, digs = eng.didx_parse(didx)
    ends = [int(x) for x in ends]
    starts = [0] + ends[:-1]
    bad = 2
    ranges = [(starts[c], ends[c] - starts[c]) for c in range(len(ends))]
    blobs = {c: store[bytes(digs[c])] for c in range(len(ends))}
    b = bytearray(blobs[bad])
    b[len(b) // 2] ^= 0x40
    blobs[bad] = bytes(b)
    bound = [E.deflate_bound(n) for _, n in ranges]
    oo = np.concatenate([[0], np.cumsum(bound)[:-1]]).astype(np.uint64)
    out = np.full(int(sum(bound)), SENT, np.uint8)
    with eng.reader(didx) as r:
        st, olen, crc, bst = raw_read_deflate(eng, r, *zip(*ranges), blobs, out, oo)
    assert bst[bad] != _lib.DEC_OK and all(bst[c] == _lib.DEC_OK for c in range(len(ends)) if c != bad)
    for c, (o, n) in enumerate(ranges):
        seg = out[int(oo[c]):int(oo[c]) + bound[c]]
        if c == bad:
            assert st[c] == bst[bad] and olen[c] == 0 and crc[c] == 0 and (seg == SENT).all()
        else:
            assert st[c] == _lib.DEC_OK and inflate(seg[:int(olen[c])].tobytes()) == archive[o:o + n]
            assert crc[c] == zlib.crc32(archive[o:o + n])


def test_a_call_that_decodes_in_groups(eng):
    files = [content(3_000_000, 900)]
    didx, offs, archive, store = write_snapshot(eng, files, "z")
    ends = [int(x) for x in eng.didx_parse(didx)[0]]
    # the cache raised to the largest chunk: every blob past the first few is decoded in a group of its own
    with transfer.PayloadReader(eng, didx, store.__getitem__, cache_bytes=1) as r:
        cuts = [0] + ends[3:len(ends):4] + [len(archive)]
        streams, _ = r._read_deflate(cuts[:-1], list(np.diff(cuts)), False)
        assert b"".join(inflate(s) for s in streams) == archive


class Zeros(io.RawIOBase):
    """n zero bytes, read in pieces (never held at once)."""

    def __init__(self, n):
        self.left = n

    def readable(self):
        return True

    def readinto(self, b):
        k = min(len(b), self.left)
        b[:k] = bytes(k)
        self.left -= k
        return k


def test_zip_writer_end_to_end(eng, tmp_path):
    rng = np.random.default_rng(17)
    big = np.tile(np.frombuffer(content(4 << 20, 901), np.uint8), 256)   # 1 GiB
    big[::4099] = rng.integers(0, 256, len(big[::4099]), dtype=np.uint8)
    tree = [("a/empty.txt", b""), ("a/b/ünïcödé ☃.txt", content(70_000, 902)), ("a/small.bin", content(5, 903)),
            ("a/big.bin", big.tobytes()), ("a/mid.txt", content(3_000_000, 904))]
    store = {}
    w = transfer.PayloadStreamWriter(eng, pg.make_config(4 << 20), upload_blob=lambda d, b: store.setdefault(d, b),
                                     blob_compression="lzh")
    offs = [w.WriteEntryReader(transfer.Entry(p, len(d)), io.BytesIO(d), len(d)) for p, d in tree]
    w.Finish()
    mt = 1_700_000_000
    zpath = tmp_path / "restore.zip"
    with transfer.PayloadReader(eng, w.didx(), store.__getitem__) as r, open(zpath, "wb") as f:
        z = transfer.ZipWriter(r, f, piece_bytes=256 << 20)
        z.AddDirectory("a", stat.S_IFDIR | 0o755, mt)
        z.AddDirectory("a/b", stat.S_IFDIR | 0o700, mt + 2)
        z.AddDirectory("a/empty-dir", stat.S_IFDIR | 0o750, mt + 4)
        z.AddFiles([(p, stat.S_IFREG | 0o640, mt + 10 * k, o, len(d)) for k, ((p, d), o) in enumerate(zip(tree, offs))])
        z.AddSymlink("a/link", "b/ünïcödé ☃.txt", stat.S_IFLNK | 0o777, mt + 6)
        z.Close()
    out = tmp_path / "x"
    with zipfile.ZipFile(zpath) as zf:
        zf.extractall(out)
        info = {i.filename: i for i in zf.infolist()}
    for k, (p, d) in enumerate(tree):
        assert (out / p).read_bytes() == d, p
        i = info[p]
        assert i.external_attr >> 16 == stat.S_IFREG | 0o640 and i.compress_type == zipfile.ZIP_DEFLATED
        assert int.from_bytes(i.extra[5:9], "little") == mt + 10 * k
    assert (out / "a/empty-dir").is_dir() and info["a/empty-dir/"].external_attr >> 16 == stat.S_IFDIR | 0o750
    assert stat.S_ISLNK(info["a/link"].external_attr >> 16)
    with zipfile.ZipFile(zpath) as zf:
        assert zf.read("a/link") == "b/ünïcödé ☃.txt".encode()
    assert info["a/big.bin"].compress_size < len(big)


def test_a_file_of_4_gib_plus_1_zeros_in_pieces(eng, tmp_path):
    size = (4 << 30) + 1
    store = {}
    w = transfer.PayloadStreamWriter(eng, pg.make_config(4 << 20), upload_blob=lambda d, b: store.setdefault(d, b),
                                     blob_compression="lzh")
    off = w.WriteEntryReader(transfer.Entry("zeros", size), io.BufferedReader(Zeros(size), 64 << 20), size)
    w.Finish()
    zpath = tmp_path / "zeros.zip"
    with transfer.PayloadReader(eng, w.didx(), store.__getitem__) as r, open(zpath, "wb") as f:
        z = transfer.ZipWriter(r, f)
        z.AddFiles([("zeros.bin", stat.S_IFREG | 0o644, 1_700_000_000, off, size)])
        z.Close()
    with zipfile.ZipFile(zpath) as zf:
        i = zf.getinfo("zeros.bin")
        assert i.file_size == size and i.compress_size < size // 100
        assert zf.testzip() is None
    assert os.path.getsize(zpath) < size // 100
