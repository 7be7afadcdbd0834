"""The sparse image restore on the GPU (pbsgpu_reader_read_sparse, K17 + K14; plan with PBSGPU_READ_SPARSE;
transfer.restore_image): extents and packed bytes equal tests/sparse_ref.py for 4 KiB, 64 KiB and 4 MiB chunks, for
images that mix zero chunks, data chunks with zero blocks and zero runs across chunk boundaries, plain and keyed, over
many, unaligned and empty ranges; zero chunks are never planned, fetched or cached; a corrupt blob fails only its
ranges and leaves their output untouched; argument errors; the restore into a file and its holes."""
import ctypes as C
import errno
import os
import random

import numpy as np
import pytest

import crypt_ref
import sparse_ref
import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib, transfer
from pbs_plus_b200.engine import _blob_args, _ptr

pytestmark = pytest.mark.gpu
KEY = bytes(range(7, 39))
B = sparse_ref.BLOCK


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


def chunk_bytes(kind: str, n: int, rng: np.random.Generator) -> np.ndarray:
    """Z: zeros.  D: random.  H: random with zero blocks and runs at several offsets -- aligned blocks, an unaligned
    run, and a zero head and tail that join the zeros of the neighbouring chunks."""
    if kind == "Z":
        return np.zeros(n, np.uint8)
    a = rng.integers(0, 256, n, dtype=np.uint8)
    if kind == "H":   # a chunk of one block keeps data between its zero runs
        runs = (((0, B), (n // 4, max(B, n // 8)), (100, 5000), (n // 2 + 7, 3 * B), (n - B - 3, B + 3)) if n >= 8 * B
                else ((100, 1000), (n - 500, 500)))
        for lo, ln in runs:
            a[lo:lo + ln] = 0
    return a


def make_image(cs: int, kinds: str, seed: int, last: int = 0) -> bytes:
    """One chunk per letter of kinds; with last, a short last chunk of that many zero bytes."""
    rng = np.random.default_rng(seed)
    parts = [chunk_bytes(k, cs, rng) for k in kinds] + ([np.zeros(last, np.uint8)] if last else [])
    return np.concatenate(parts).tobytes()


def write_image(eng, data: bytes, cs: int, mode: str, key: bytes | None):
    """-> (.fidx, {digest: blob}).  "raw" blobs come from the encrypted batch encoder (the writer compresses)."""
    if mode == "raw":
        a = np.frombuffer(data, np.uint8)
        off = np.arange(0, len(data), cs, dtype=np.uint64)
        ln = np.minimum(np.uint64(len(data)) - off, np.uint64(cs))
        crypt = eng.crypt(key)
        dig = eng.sha256_keyed_batch(crypt, a, off, ln)
        blobs = eng.blob_encode_batch_enc(crypt, "raw", a, off, ln, os.urandom(16 * len(off)))[0]
        crypt.close()
        return eng.fidx_build(dig, len(data), cs), {bytes(d): b for d, b in zip(dig, blobs)}
    store = {}
    w = transfer.FixedIndexWriter(eng, cs, eng.digest_set(), upload_blob=store.__setitem__, blob_compression=mode,
                                  crypt_key=key)
    w.WriteSlice(data)
    return w.fidx(), store


def zero_chunks(eng, fidx: bytes, key: bytes | None) -> set[int]:
    size, cs, dig = eng.fidx_parse(fidx)
    ident = crypt_ref.id_key(key) if key else None
    return {c for c in range(len(dig))
            if bytes(dig[c]) == sparse_ref.zero_digest(min(cs, size - c * cs), ident)}


def touched(off: int, length: int, cs: int) -> set[int]:
    return set(range(off // cs, (off + length - 1) // cs + 1)) if length else set()


def check(data: bytes, ranges, status, got) -> None:
    assert status.tolist() == [0] * len(ranges)
    for (o, l), g in zip(ranges, got):
        ext = sparse_ref.extents(data, o, l)
        assert g == (ext, sparse_ref.packed(data, ext)), (o, l)


def random_ranges(size: int, n: int, seed: int, cs: int):
    rng = random.Random(seed)
    out = [(0, size), (0, 0), (size, 0), (size - 1, 1), (B - 1, 2), (cs - 1, 2)]
    for _ in range(n):
        a = rng.randrange(0, size + 1)
        out.append((a, rng.randrange(0, min(size - a, 3 * cs) + 1)))
    return out


CASES = [(4 << 10, "lzh", None), (64 << 10, "lzh", None), (4 << 20, "lzh", None), (64 << 10, "z", None),
         (64 << 10, "raw", KEY), (64 << 10, "lzh", KEY)]


@pytest.mark.parametrize("cs,mode,key", CASES, ids=[f"{cs >> 10}k-{m}-{'key' if k else 'plain'}" for cs, m, k in CASES])
def test_read_sparse_equals_the_restatement(eng, cs, mode, key):
    kinds = "ZZDHZHHZDZZZHDZZ" if cs >= 4 << 20 else "ZZDHZHHZDZZZHDZZ" * 3
    data = make_image(cs, kinds, cs + len(mode), last=cs // 2 + 1234 if cs > 4096 else 1234)
    fidx, store = write_image(eng, data, cs, mode, key)
    zeros = zero_chunks(eng, fidx, key)
    assert zeros == {c for c, k in enumerate(kinds) if k == "Z"} | {len(kinds)}   # the short last chunk is zero too
    size = len(data)
    ranges = random_ranges(size, 40, cs, cs)
    offs, lens = [a for a, _ in ranges], [b for _, b in ranges]
    crypt = eng.crypt(key) if key else None
    with eng.reader_fidx(fidx, crypt, cache_bytes=64 * cs) as r:
        # many ranges in one call: the sparse plan names exactly the data chunks they touch, the plain plan all
        want = set().union(*(touched(a, b, cs) for a, b in ranges))
        chunks, dig = r.plan(offs, lens, sparse=True)
        assert chunks.tolist() == sorted(want - zeros)
        assert r.plan(offs, lens)[0].tolist() == sorted(want)
        st, got, bst = r.read_sparse(offs, lens, {int(c): store[bytes(d)] for c, d in zip(chunks, dig)})
        assert (bst == 0).all()
        check(data, ranges, st, got)
        # range by range, from the cache where it still holds them; zero chunks never need a blob
        for o, l in ranges[:12] + [(c * cs, cs) for c in sorted(zeros)[:3]]:
            chunks, dig = r.plan([o], [l], sparse=True)
            st, got, _ = r.read_sparse([o], [l], {int(c): store[bytes(d)] for c, d in zip(chunks, dig)})
            check(data, [(o, l)], st, got)
    if crypt is not None:
        crypt.close()


def raw_read_sparse(r, off, length, blobs, out, ext_cap=None, flags=0):
    """pbsgpu_reader_read_sparse through ctypes with a caller-filled out -> (rc, status, ext pairs, ext_first, bst)."""
    o, l = pg.Engine._offlen(off, length)
    base, bo, bl, bc = _blob_args(blobs)
    n, k = len(o), len(bo)
    oo = np.zeros(n, np.uint64)
    oo[1:] = np.cumsum(l)[:-1]
    bound = sum(sparse_ref.ext_bound(int(a), int(b)) for a, b in zip(o, l))
    cap = bound if ext_cap is None else ext_cap
    ext = np.full((cap + 4, 2), 0xEEEE, np.uint64)   # 4 sentinel pairs past the capacity the call is given
    first = np.zeros(n + 1, np.uint64)
    st, bst = np.zeros(n, np.int32), np.zeros(k, np.int32)
    rc = r._eng._L.pbsgpu_reader_read_sparse(r._h, o.ctypes.data, l.ctypes.data, n, flags, _ptr(base), bo.ctypes.data,
                                             bl.ctypes.data, bc.ctypes.data, k, _ptr(out), oo.ctypes.data, ext.ctypes.data,
                                             cap, first.ctypes.data, st.ctypes.data, bst.ctypes.data)
    assert (ext[cap:] == 0xEEEE).all(), "extents written past ext_cap"
    return rc, st, ext[:cap], first, bst, oo


def test_a_two_chunk_cache_restores_hundreds_of_zero_chunks(eng):
    """A cache of two 4 KiB chunks and an image of 2 data chunks among 400 zero chunks: one call, no eviction, and the
    data chunks are still cached for the next call -- no zero chunk took a slot."""
    cs = 4 << 10
    kinds = "Z" * 150 + "D" + "Z" * 200 + "H" + "Z" * 50
    data = make_image(cs, kinds, 5)
    fidx, store = write_image(eng, data, cs, "lzh", None)
    with eng.reader_fidx(fidx, cache_bytes=2 * cs) as r:
        chunks, dig = r.plan([0], [len(data)], sparse=True)
        assert chunks.tolist() == [150, 351]
        st, got, bst = r.read_sparse([0], [len(data)], {int(c): store[bytes(d)] for c, d in zip(chunks, dig)})
        check(data, [(0, len(data))], st, got)
        assert r.plan([0], [len(data)], sparse=True)[0].tolist() == []
        assert r.plan([0], [len(data)])[0].tolist() == [c for c, k in enumerate(kinds) if k == "Z"]
        st, got, _ = r.read_sparse([0, 150 * cs + 9], [len(data), 250 * cs], {})
        check(data, [(0, len(data)), (150 * cs + 9, 250 * cs)], st, got)


def test_corrupt_blob_fails_only_its_ranges(eng):
    cs = 64 << 10
    kinds = "DZHDZZDH"
    data = make_image(cs, kinds, 9, last=777)
    fidx, store = write_image(eng, data, cs, "lzh", None)
    _, _, dig = eng.fidx_parse(fidx)
    blobs = {c: store[bytes(dig[c])] for c in range(len(dig))}   # zero chunks' blobs too: checked, not needed
    bad = bytearray(blobs[3]); bad[-1] ^= 0x40; blobs[3] = bytes(bad)
    ranges = [(0, 3 * cs), (2 * cs + 5, 2 * cs), (3 * cs + 100, 1), (4 * cs, len(data) - 4 * cs), (0, 0), (cs, cs)]
    with eng.reader_fidx(fidx) as r:
        total = sum(b for _, b in ranges)
        out = np.full(max(1, total), 0xA5, np.uint8)
        rc, st, ext, first, bst, oo = raw_read_sparse(r, [a for a, _ in ranges], [b for _, b in ranges], blobs, out)
        assert rc == 0
        assert st.tolist() == [0, _lib.DEC_BAD_CRC, _lib.DEC_BAD_CRC, 0, 0, 0]
        assert bst.tolist() == [_lib.DEC_BAD_CRC if c == 3 else 0 for c in range(len(dig))]
        for i, (a, b) in enumerate(ranges):
            e = [(int(x), int(y)) for x, y in ext[int(first[i]):int(first[i + 1])]]
            region = out[int(oo[i]):int(oo[i]) + b]
            if st[i]:
                assert e == [] and (region == 0xA5).all()
            else:
                want = sparse_ref.extents(data, a, b)
                p = sparse_ref.packed(data, want)
                assert e == want and region[:len(p)].tobytes() == p and (region[len(p):] == 0xA5).all()


def test_argument_errors_leave_the_reader_usable(eng):
    cs = 4 << 10
    data = make_image(cs, "DZHZ", 3, last=100)
    fidx, store = write_image(eng, data, cs, "z", None)
    rec = np.zeros(2, dtype=_lib.CHUNK_DTYPE)
    rec["end_off"] = [cs, 2 * cs]
    didx = eng.didx_build(rec)
    out = np.zeros(len(data), np.uint8)
    with eng.reader(didx) as d:
        assert raw_read_sparse(d, [0], [10], {}, out)[0] == _lib.EINVAL
        with pytest.raises(pg.PbsGpuError) as e:
            d.plan([0], [10], sparse=True)
        assert e.value.code == _lib.EINVAL
    with eng.reader_fidx(fidx) as r:
        ranges = ([1, B - 1, 0], [3 * B, B + 2, len(data) - 1])
        bound = sum(sparse_ref.ext_bound(a, b) for a, b in zip(*ranges))
        assert raw_read_sparse(r, *ranges, {}, out, ext_cap=bound - 1)[0] == _lib.EINVAL
        assert raw_read_sparse(r, [0], [10], {}, out, flags=_lib.READ_PAYLOAD)[0] == _lib.EINVAL
        assert raw_read_sparse(r, [0], [10], {}, out, flags=_lib.READ_SPARSE)[0] == _lib.EINVAL
        for call in (lambda f: r._eng._L.pbsgpu_reader_read(r._h, *rd_args(f, out)),
                     lambda f: r._eng._L.pbsgpu_reader_read_deflate(r._h, *rdf_args(f, out))):
            assert call(_lib.READ_SPARSE) == _lib.EINVAL
        # still usable: the same ranges with room for their extents
        chunks, dig = r.plan(*ranges, sparse=True)
        st, got, _ = r.read_sparse(*ranges, {int(c): store[bytes(x)] for c, x in zip(chunks, dig)})
        check(data, list(zip(*ranges)), st, got)


_keep = []   # the ctypes arrays of rd_args / rdf_args outlive the call


def rd_args(flags, out):
    o, l = np.zeros(1, np.uint64), np.full(1, 10, np.uint64)
    st = np.zeros(1, np.int32)
    _keep[:] = [o, l, st]
    return (o.ctypes.data, l.ctypes.data, 1, flags, None, None, None, None, 0, out.ctypes.data, o.ctypes.data,
            st.ctypes.data, None)


def rdf_args(flags, out):
    o, l = np.zeros(1, np.uint64), np.full(1, 10, np.uint64)
    olen, st = np.zeros(1, np.uint64), np.zeros(1, np.int32)
    _keep[:] = [o, l, olen, st]
    return (o.ctypes.data, l.ctypes.data, 1, flags, None, None, None, None, None, 0, out.ctypes.data, o.ctypes.data,
            olen.ctypes.data, None, st.ctypes.data, None)


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


@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "key"])
def test_restore_image_writes_only_the_data(eng, tmp_path, key):
    cs = 64 << 10
    kinds = "ZZDHZHHZDZZZHDZZ" * 2
    data = make_image(cs, kinds, 21, last=9000)
    fidx, store = write_image(eng, data, cs, "lzh", key)
    zero_digests = {sparse_ref.zero_digest(n, crypt_ref.id_key(key) if key else None) for n in (cs, 9000)}
    asked = []

    def source(d: bytes) -> bytes:
        asked.append(d)
        return store[d]

    path = tmp_path / "disk.img"
    fd = os.open(path, os.O_RDWR | os.O_CREAT | os.O_TRUNC, 0o600)
    try:
        transfer.restore_image(eng, fidx, source, fd, crypt_key=key, slice_bytes=5 * cs + 4096)
    finally:
        os.close(fd)
    assert path.read_bytes() == data
    assert asked and not zero_digests & set(asked)
    if not seek_hole_works(tmp_path):
        return   # this filesystem does not report holes; the bytes above are still checked
    fd = os.open(path, os.O_RDONLY)
    try:
        for lo, hi in sparse_ref.holes(data, len(data)):
            try:
                assert os.lseek(fd, lo, os.SEEK_DATA) >= hi, (lo, hi)
            except OSError as e:
                assert e.errno == errno.ENXIO   # no data after lo: a hole to the end
    finally:
        os.close(fd)


def test_restore_image_names_the_corrupt_chunk(eng, tmp_path):
    cs = 4 << 10
    data = make_image(cs, "DZZHD", 4)
    fidx, store = write_image(eng, data, cs, "lzh", None)
    _, _, dig = eng.fidx_parse(fidx)
    bad = bytes(dig[3])
    store[bad] = store[bad][:-1] + bytes([store[bad][-1] ^ 1])
    fd = os.open(tmp_path / "x.img", os.O_RDWR | os.O_CREAT, 0o600)
    try:
        with pytest.raises(IOError, match=f"chunk 3 \\({bad.hex()}\\)"):
            transfer.restore_image(eng, fidx, store.__getitem__, fd)
    finally:
        os.close(fd)


def write_image_any(eng, data: bytes, cs: int):
    """-> (.fidx, {digest: blob}) for any chunk size (the writers take powers of two of 4 KiB or more; an index read
    from a server may carry any size), with _lzh blobs."""
    a = np.frombuffer(data, np.uint8)
    off = np.arange(0, len(data), cs, dtype=np.uint64)
    ln = np.minimum(np.uint64(len(data)) - off, np.uint64(cs))
    dig = eng.sha256_batch(a, off, ln)
    blobs = eng.blob_encode_batch_lzh(a, off, ln)[0]
    return eng.fidx_build(dig, len(data), cs), {bytes(d): b for d, b in zip(dig, blobs)}


ODD = [(1000, "DZDZD", 0), (6144, "DZD", 0), (6144, "DZZDHZZZ", 3000), (10240, "DZZDHZ", 3000), (4097, "ZDZZHDZ", 17)]


@pytest.mark.parametrize("cs,kinds,last", ODD, ids=[f"{cs}-{k}" for cs, k, _ in ODD])
def test_chunk_sizes_that_cut_blocks(eng, tmp_path, cs, kinds, last):
    """An index whose chunk size is not a multiple of 4096: a zero chunk that shares a block with a data chunk is read
    like a data chunk, so every block part with a data byte is one piece of one extent, the extents still equal the
    restatement and fit the ceil(B / 2) bound (the sentinel pairs past ext_cap stay untouched); zero chunks on block
    boundaries, such as a short last chunk that starts on one, are still served by digest."""
    data = make_image(cs, kinds, cs, last=last)
    size = len(data)
    fidx, store = write_image_any(eng, data, cs)
    zeros = zero_chunks(eng, fidx, None)
    served = {c for c in zeros if sparse_ref.served_by_digest(c * cs, min((c + 1) * cs, size), size)}
    ranges = random_ranges(size, 30, cs, cs) + [(0, min(size, 4 * B)), (B - 5, min(2 * B + 9, size - B + 5))]
    offs, lens = [a for a, _ in ranges], [b for _, b in ranges]
    with eng.reader_fidx(fidx) as r:
        want = set().union(*(touched(a, b, cs) for a, b in ranges))
        chunks, dig = r.plan(offs, lens, sparse=True)
        assert chunks.tolist() == sorted(want - served)
        blobs = {int(c): store[bytes(d)] for c, d in zip(chunks, dig)}
        out = np.full(max(1, sum(lens)), 0xA5, np.uint8)
        rc, st, ext, first, _, oo = raw_read_sparse(r, offs, lens, blobs, out)
        assert rc == 0 and st.tolist() == [0] * len(ranges)
        for i, (a, b) in enumerate(ranges):
            want_ext = sparse_ref.extents(data, a, b)
            assert [(int(x), int(y)) for x, y in ext[int(first[i]):int(first[i + 1])]] == want_ext, (a, b)
            p = sparse_ref.packed(data, want_ext)
            assert out[int(oo[i]):int(oo[i]) + len(p)].tobytes() == p, (a, b)
    path = tmp_path / "odd.img"
    fd = os.open(path, os.O_RDWR | os.O_CREAT | os.O_TRUNC, 0o600)
    try:
        transfer.restore_image(eng, fidx, store.__getitem__, fd, slice_bytes=3 * cs)
    finally:
        os.close(fd)
    assert path.read_bytes() == data
