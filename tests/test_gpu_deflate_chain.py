"""pbsgpu_deflate_batch_lzc on the GPU (K16's DEFLATE instantiation + K15): byte-identical to tests/deflate_chain_ref.py
on every CPU case, from host and ragged device bases into host and device out; pieces joined through `more`; a call
over more than one pass; 256 MiB of each corpus inflates through zlib and is smaller than pbsgpu_deflate_batch's stream;
the bound on random data; pbsgpu_reader_read_deflate with PBSGPU_READ_DEFLATE_LZC equal to the batch call, plain and
encrypted, a corrupt blob failing only its own ranges, plan and read refusing the flag; and ZipWriter(lzc=True)."""
import ctypes
import io
import stat
import zipfile
import zlib

import numpy as np
import pytest

import deflate_chain_ref as ch
import deflate_ref as dr
import pbs_plus_b200 as pg
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from pbs_plus_b200 import _lib, engine as E, transfer
from pbs_plus_b200._lib import EINVAL
from test_deflate_chain_cpu import cases
from test_gpu_deflate import half_zero_random, pack
from test_gpu_reader import KEY, SENT, content, write_snapshot
from test_gpu_zip import raw_read_deflate

pytestmark = pytest.mark.gpu
SEG = dr.SEGMENT
LZC = _lib.READ_DEFLATE_LZC


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def ref():
    cs = cases()
    return list(cs), [cs[k] for k in cs], [ch.deflate(cs[k]) for k in cs]


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("out", ["host", "device"])
def test_byte_identical_to_the_restatement(eng, torch, ref, where, out):
    names, parts, want = ref
    buf, off, ln = pack(parts, 5 if where == "device" else 0)
    base = torch.from_numpy(buf).cuda() if where == "device" else buf
    got, crc = eng.deflate_batch_lzc(base, off, ln, out=out)
    for k, name in enumerate(names):
        g = got[k] if out == "host" else got[k].cpu().numpy().tobytes()
        assert g == want[k], name
        assert crc[k] == zlib.crc32(parts[k]), name


def test_pieces_through_more(eng, torch):
    data = lzref.text_corpus(5 * SEG + 999, 21).tobytes()
    whole = ch.deflate(data)
    dev = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).cuda()
    cuts = [0, SEG, 3 * SEG, len(data)]
    got, crc = eng.deflate_batch_lzc(dev, np.array(cuts[:-1], np.uint64), np.diff(np.array(cuts, np.uint64)),
                                     more=[1, 1, 0])
    assert b"".join(got) == whole and zlib.decompress(whole, -15) == data
    c = int(crc[0])
    for k in (1, 2):
        c = pg.engine.crc32_combine(c, int(crc[k]), cuts[k + 1] - cuts[k])
    assert c == zlib.crc32(data)
    with pytest.raises(pg.PbsGpuError) as e:
        eng.deflate_batch_lzc(dev, [0], [SEG + 1], more=[1])
    assert e.value.code == EINVAL
    got, _ = eng.deflate_batch_lzc(dev, [0, 0], [0, 0], more=[1, 0])
    assert got == [b"", b"\x03\x00"]


def test_a_call_over_more_than_one_pass(eng, torch):
    """2085 ranges of about one segment, ragged, and two of six segments that straddle the pass edges at segment 1024
    and 2048 (one pass is DCH_PASS_SEGS = 1024 segments): all inflate, and the ranges next to both edges equal the
    restatement."""
    nr = 2085
    ln = [SEG - k % 5 for k in range(nr)]
    ln[1022] = ln[2040] = 5 * SEG + 3
    off = np.concatenate([[0], np.cumsum(np.array(ln) + 7)[:-1]]).astype(np.uint64)   # 7 bytes apart
    total = int(off[-1]) + ln[-1]
    a = np.concatenate([lzref.text_corpus(total // 2, 22), hufref.binary_corpus(total - total // 2, 23)])
    dev = torch.from_numpy(a).cuda()
    got, crc = eng.deflate_batch_lzc(dev, off, np.array(ln, np.uint64))
    greedy, _ = eng.deflate_batch(dev, off, np.array(ln, np.uint64))
    for k in range(nr):
        piece = a[int(off[k]):int(off[k]) + ln[k]].tobytes()
        assert zlib.decompress(got[k], -15) == piece and crc[k] == zlib.crc32(piece), k
    assert sum(map(len, got)) < sum(map(len, greedy))
    for k in (0, 1021, 1022, 1023, 2039, 2040, 2041, nr - 1):
        assert got[k] == ch.deflate(a[int(off[k]):int(off[k]) + ln[k]].tobytes()), k


def test_bound_on_random_data(eng, torch):
    rng = np.random.default_rng(31)
    parts = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (1, 77, 65535, SEG, 3 * SEG + 5, 9 << 20)]
    buf, off, ln = pack(parts, 0)
    got, crc = eng.deflate_batch_lzc(torch.from_numpy(buf).cuda(), off, ln)
    for p, g, c in zip(parts, got, crc):
        assert len(g) <= pg.engine.deflate_bound(len(p)) and zlib.decompress(g, -15) == p and c == zlib.crc32(p)


@pytest.mark.parametrize("corpus", ["half_zero_random", "text", "binary"])
def test_256_mib_inflates_and_is_smaller_than_greedy(eng, torch, corpus):
    n = 256 << 20
    a = {"half_zero_random": lambda: half_zero_random(n, 1), "text": lambda: lzref.text_corpus(n, 2),
         "binary": lambda: hufref.binary_corpus(n, 3)}[corpus]()
    dev = torch.from_numpy(a).cuda()
    cut = [0, n // 3 + 1, 2 * n // 3 + 7, n]                 # three ranges, ragged ends
    off, ln = np.array(cut[:-1], np.uint64), np.diff(np.array(cut, np.uint64))
    got, crc = eng.deflate_batch_lzc(dev, off, ln, out="device")
    greedy, _ = eng.deflate_batch(dev, off, ln, out="device")
    for i in range(3):
        s = got[i].cpu().numpy().tobytes()
        piece = a[cut[i]:cut[i + 1]].tobytes()
        assert zlib.decompress(s, -15) == piece and crc[i] == zlib.crc32(piece)
        assert len(s) < len(greedy[i])


# ---- the reader ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "encrypted"])
def test_read_deflate_lzc_equals_the_batch_call(eng, key):
    files = [content(n, 1700 + i) for i, n in enumerate([0, 1, 5000, 200_000, 3 * SEG + 17, 700_000])]
    didx, offs, archive, store = write_snapshot(eng, files, "lzh", key)
    sizes = [len(f) for f in files]
    a = np.frombuffer(archive, np.uint8)
    want, wcrc = eng.deflate_batch_lzc(a, [o + 16 for o in offs], sizes)
    with transfer.PayloadReader(eng, didx, store.__getitem__, crypt_key=key) as r:
        streams, crcs = r._read_deflate(offs, sizes, True, None, True)
        assert streams == want and crcs == [int(c) for c in wcrc]
        assert [zlib.decompress(s, -15) for s in streams] == files
        greedy, _ = r._read_deflate(offs, sizes, True)
        assert greedy == eng.deflate_batch(a, [o + 16 for o in offs], sizes)[0]
        # plain ranges with pieces continued by `more`
        lo = offs[4] + 16
        st, got, crc, _ = r._reader.read_deflate([lo, lo + SEG], [SEG, 2 * SEG + 17], r._fetch([lo], [3 * SEG + 17], False),
                                                 False, [1, 0], True)
        assert list(st) == [_lib.DEC_OK] * 2 and b"".join(got) == ch.deflate(files[4])


def test_a_corrupt_blob_fails_only_its_ranges(eng):
    files = [content(n, 1800 + i) for i, n in enumerate([200_000, 300_000, 150_000])]
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
    a = np.frombuffer(archive, np.uint8)
    with eng.reader(didx) as r:
        st, olen, crc, bst = raw_read_deflate(eng, r, *zip(*ranges), blobs, out, oo, flags=LZC)
    assert bst[bad] != _lib.DEC_OK
    for c, (o, n) in enumerate(ranges):
        seg = out[int(oo[c]):int(oo[c]) + bound[c]]
        if c == bad:
            assert st[c] == bst[bad] and olen[c] == 0 and crc[c] == 0 and (seg == SENT).all()
        else:
            assert st[c] == _lib.DEC_OK
            assert seg[:int(olen[c])].tobytes() == eng.deflate_batch_lzc(a, [o], [n])[0][0]


def test_plan_and_read_refuse_the_flag(eng):
    files = [content(100_000, 1900)]
    didx, offs, archive, store = write_snapshot(eng, files, "z")
    o, l = np.array([offs[0]], np.uint64), np.array([len(files[0])], np.uint64)
    chunk = np.zeros(64, np.uint64)
    n_out = ctypes.c_uint64(0)
    out = np.zeros(len(files[0]) + 64, np.uint8)
    oo, st = np.zeros(1, np.uint64), np.zeros(1, np.int32)
    with eng.reader(didx) as r:
        for flags in (LZC, LZC | _lib.READ_PAYLOAD):
            assert eng._L.pbsgpu_reader_plan(r._h, o.ctypes.data, l.ctypes.data, 1, flags, chunk.ctypes.data, None, 64,
                                             ctypes.byref(n_out)) == EINVAL
            assert eng._L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, 1, flags, None, None, None, None, 0,
                                             out.ctypes.data, oo.ctypes.data, st.ctypes.data, None) == EINVAL


def test_zip_writer_lzc(eng, tmp_path):
    tree = [("t/a.txt", lzref.text_corpus(3_000_000, 31).tobytes()), ("t/b.bin", hufref.binary_corpus(700_000, 32).tobytes()),
            ("t/empty", b""), ("t/c.txt", content(90_000, 33))]
    store = {}
    w = transfer.PayloadStreamWriter(eng, pg.make_config(1 << 20), upload_blob=lambda d, b: store.setdefault(d, b),
                                     blob_compression="lzh")
    offs = [w.WriteEntryReader(transfer.Entry(p, len(d)), io.BytesIO(d), len(d)) for p, d in tree]
    w.Finish()
    sizes = {}
    for lzc in (False, True):
        zpath = tmp_path / f"r{int(lzc)}.zip"
        with transfer.PayloadReader(eng, w.didx(), store.__getitem__) as r, open(zpath, "wb") as f:
            z = transfer.ZipWriter(r, f, piece_bytes=1 << 20, lzc=lzc)   # t/a.txt goes in pieces
            z.AddFiles([(p, stat.S_IFREG | 0o644, 1_700_000_000, o, len(d)) for (p, d), o in zip(tree, offs)])
            z.Close()
        with zipfile.ZipFile(zpath) as zf:
            assert zf.testzip() is None
            assert all(zf.read(p) == d for p, d in tree)
        sizes[lzc] = zpath.stat().st_size
    assert sizes[True] < sizes[False]
