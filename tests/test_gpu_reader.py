"""The archive reader on the GPU (pbsgpu_reader_*: K6 / K11 / K13 / K3 into a device cache, K14 out of it): payload
streams written by PayloadStreamWriter in every mode, plain and encrypted, read back byte-exactly by file and by
arbitrary range, also across WriteEntryRef; the FIFO cache, its groups and prefetch; every status between intact
neighbours with no byte of a failed chunk in the output; host and device outputs and blob bases; lifecycle and argument
errors."""
import ctypes as C
import hashlib
import io
import os
import random

import numpy as np
import pytest

import pbs_plus_b200 as pg
import zstd_lz_ref as lzref
from pbs_plus_b200 import _lib, transfer
from pbs_plus_b200.engine import _ptr

pytestmark = pytest.mark.gpu
AVG = 1 << 16
KEY = bytes(range(7, 39))
SENT = 0xA5


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


def content(n: int, seed: int) -> bytes:
    """Text, zero runs and random bytes, so every mode writes compressed and raw blocks."""
    rng = np.random.default_rng(seed)
    parts = [lzref.text_corpus(n, seed), np.zeros(n, np.uint8), rng.integers(0, 256, n, dtype=np.uint8)]
    pick = rng.integers(0, 3, n // 4096 + 1)
    out = np.concatenate([parts[p][k * 4096:(k + 1) * 4096] for k, p in enumerate(pick)])[:n]
    return out.tobytes()


def file_sizes(cfg) -> list[int]:
    rng = random.Random(5)
    edges = [int(cfg.min) - 1, int(cfg.min), AVG, int(cfg.max), int(cfg.max) + 1]
    return [0, 1, *edges, 3 * int(cfg.max) + 12345] + [rng.randrange(2, 200_000) for _ in range(12)]


def marker(m: int) -> bytes:
    return m.to_bytes(8, "little") + (16).to_bytes(8, "little")


def write_snapshot(eng, files, mode="lzh", key=None, store=None):
    """A payload stream of `files` into `store` (digest -> blob) -> (didx, payload offsets, archive bytes, store)."""
    store = {} if store is None else store
    w = transfer.PayloadStreamWriter(eng, pg.make_config(AVG), upload_blob=lambda d, b: store.setdefault(d, b),
                                     blob_compression=mode, crypt_key=key)
    offs = [w.WriteEntryReader(transfer.Entry(f"f{i}", len(f)), io.BytesIO(f), len(f)) for i, f in enumerate(files)]
    w.Finish()
    archive = marker(transfer.PXAR_PAYLOAD_START_MARKER) + b"".join(transfer.payload_header(len(f)) + f for f in files) \
        + marker(transfer.PXAR_PAYLOAD_TAIL_MARKER)
    return w.didx(), offs, archive, store


def manual_archive(eng, data: bytes, ends, mode="z", crypt=None):
    """An index with the chunk ends given (zero-length chunks allowed) and the blobs of its chunks by index."""
    a = np.frombuffer(data, np.uint8)
    e = np.array(ends, np.uint64)
    off = np.concatenate([[0], e[:-1]]).astype(np.uint64)
    ln = e - off
    if crypt is not None:
        dig = eng.sha256_keyed_batch(crypt, a, off, ln)
        blobs = eng.blob_encode_batch_enc(crypt, mode, a, off, ln, os.urandom(16 * len(e)))[0]
    else:
        dig = eng.sha256_batch(a, off, ln)
        blobs = getattr(eng, "blob_encode_batch_" + mode)(a, off, ln)[0]
    rec = np.zeros(len(e), dtype=_lib.CHUNK_DTYPE)
    rec["end_off"] = e
    rec["digest"] = dig
    return eng.didx_build(rec), blobs


def raw_read(eng, r, off, ln, blobs: dict, out, out_off, flags=0):
    """pbsgpu_reader_read into the caller's `out` (filled with SENT by the caller) -> (status, blob_status)."""
    o, l = np.array(off, np.uint64), np.array(ln, np.uint64)
    oo = np.array(out_off, np.uint64)
    items = list(blobs.items())
    bc = np.array([c for c, _ in items], np.uint64)
    bl = np.array([len(b) for _, b in items], np.uint64)
    bo = np.concatenate([[0], np.cumsum(bl)[:-1]]).astype(np.uint64) if items else np.zeros(0, np.uint64)
    base = np.frombuffer(b"".join(b for _, b in items) or b"\0", np.uint8)
    st = np.full(len(o), -1, np.int32)
    bst = np.full(len(items), -1, np.int32)
    eng._ck(eng._L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, len(o), flags, base.ctypes.data, bo.ctypes.data,
                                      bl.ctypes.data, bc.ctypes.data, len(items), _ptr(out), oo.ctypes.data, st.ctypes.data,
                                      bst.ctypes.data))
    return st, bst


# ---- 1. round trips -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", [None, KEY], ids=["plain", "encrypted"])
@pytest.mark.parametrize("mode", ["z", "lzh", "lzl"])
def test_files_and_ranges_read_back_byte_exactly(eng, mode, key):
    cfg = pg.make_config(AVG)
    files = [content(n, 100 + i) for i, n in enumerate(file_sizes(cfg))]
    didx, offs, archive, store = write_snapshot(eng, files, mode, key)
    ends, _ = eng.didx_parse(didx)
    ends = [int(x) for x in ends]
    assert ends[-1] == len(archive) and len(ends) > 12
    with transfer.PayloadReader(eng, didx, store.__getitem__, crypt_key=key) as r:
        assert r.Size == len(archive)
        assert r.ReadFileContents(list(zip(offs, [len(f) for f in files]))) == files
        size = len(archive)
        for off, n in [(ends[2] + 10, 100), (ends[3] - 50, 100), (ends[1] + 5, ends[9] - ends[1]), (1234, 0), (0, size),
                       (size - 777, 777), (size - 100, 1000), (size, 10), (ends[0], ends[1] - ends[0])]:
            assert r.ReadAt(off, n) == archive[off:off + n], (off, n)
        assert r.ReadAt(size + 5, 10) == b""
        assert r.ReadFileContents([]) == []


def test_write_entry_ref_snapshot_reads_from_the_shared_store(eng):
    files = [content(n, 200 + i) for i, n in enumerate([300_000, 150_000, 500_000, 20_000])]
    didx0, offs0, _, store = write_snapshot(eng, files, "lzh", KEY)
    ends, digs = eng.didx_parse(didx0)
    w = transfer.PayloadStreamWriter(eng, pg.make_config(AVG), prev_index=(ends, digs), crypt_key=KEY,
                                     upload_blob=lambda d, b: store.setdefault(d, b), blob_compression="lzh")
    new = content(250_000, 300)
    o_new = w.WriteEntryReader(transfer.Entry("new", len(new)), io.BytesIO(new), len(new))
    o1 = w.WriteEntryRef(transfer.Entry("f1", len(files[1])), offs0[1])
    o2 = w.WriteEntryRef(transfer.Entry("f2", len(files[2])), offs0[2])
    o_end = w.WriteEntryReader(transfer.Entry("end", 1000), io.BytesIO(new[:1000]), 1000)
    w.Finish()
    with transfer.PayloadReader(eng, w.didx(), store.__getitem__, crypt_key=KEY) as r:
        got = r.ReadFileContents([(o_new, len(new)), (o1, len(files[1])), (o2, len(files[2])), (o_end, 1000)])
    assert got == [new, files[1], files[2], new[:1000]]


# ---- 3. the cache ---------------------------------------------------------------------------------------------
def test_plan_read_and_a_second_read_without_blobs(eng):
    files = [content(n, 400 + i) for i, n in enumerate([90_000, 400_000, 3, 250_000])]
    didx, offs, archive, store = write_snapshot(eng, files, "lzh")
    ends, digs = eng.didx_parse(didx)
    off = [int(ends[1]) - 7, 5, int(ends[4]) + 3]
    ln = [int(ends[5]) - off[0], 20, 40_000]
    with eng.reader(didx) as r:
        chunks, dg = r.plan(off, ln)
        assert list(chunks) == sorted(set(chunks.tolist())) and (np.diff(chunks.astype(np.int64)) > 0).all()
        assert (dg == digs[chunks.astype(np.int64)]).all()
        st, data, bst = r.read(off, ln, {int(c): store[bytes(d)] for c, d in zip(chunks, dg)})
        assert (st == _lib.DEC_OK).all() and (bst == _lib.DEC_OK).all()
        assert data == [archive[o:o + n] for o, n in zip(off, ln)]
        assert len(r.plan(off, ln)[0]) == 0
        st, data, bst = r.read(off, ln, {})
        assert (st == _lib.DEC_OK).all() and len(bst) == 0 and data == [archive[o:o + n] for o, n in zip(off, ln)]
        # the payload form over the same cache
        files_rng = [(o, len(f)) for o, f in zip(offs, files)]
        need, dg = r.plan(*zip(*files_rng), payload=True)
        st, data, _ = r.read(*zip(*files_rng), {int(c): store[bytes(d)] for c, d in zip(need, dg)}, payload=True)
        assert (st == _lib.DEC_OK).all() and data == files


def test_fifo_eviction_and_the_cache_raised_to_the_largest_chunk(eng):
    files = [content(1_500_000, 500)]
    didx, _, archive, store = write_snapshot(eng, files, "z")
    ends, digs = eng.didx_parse(didx)
    ends = [int(x) for x in ends]
    starts = [0] + ends[:-1]
    slot = [max(256, (e - s + 255) // 256 * 256) for s, e in zip(starts, ends)]
    a = int(np.argmax(slot))
    others = [c for c in range(len(ends)) if c != a][:3]
    order = [a] + others          # the fourth slot is no larger than the first: it evicts exactly the first
    blob = lambda c: {c: store[bytes(digs[c])]}
    one = lambda c: ([starts[c] + 1], [1])
    with eng.reader(didx, cache_bytes=slot[a] + slot[others[0]] + slot[others[1]]) as r:
        for c in order:
            st, data, _ = r.read(*one(c), blob(c))
            assert st[0] == _lib.DEC_OK and data[0] == archive[starts[c] + 1:starts[c] + 2]
        assert r.plan([starts[c] for c in order], [1] * 4)[0].tolist() == [a]
    with eng.reader(didx, cache_bytes=1) as r:    # raised to the largest chunk
        st, _, _ = r.read(*one(a), blob(a))
        assert st[0] == _lib.DEC_OK and len(r.plan(*one(a))[0]) == 0
        st, _, _ = r.read(*one(others[0]), blob(others[0]))
        assert st[0] == _lib.DEC_OK and r.plan(*one(a))[0].tolist() == [a]


def test_one_call_over_a_gibibyte_in_several_groups(eng, torch):
    n = 1 << 30
    g = torch.Generator(device="cuda").manual_seed(9)
    data = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=g)
    data[n // 3: n // 3 + (64 << 20)] = 0
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), data, [0], [n])
    ends = rec["end_off"].astype(np.uint64)
    off = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    blobs, _ = eng.blob_encode_batch_z(data, off, ends - off)
    didx = eng.didx_build(rec)
    base = np.frombuffer(b"".join(blobs), np.uint8)
    bl = np.array([len(b) for b in blobs], np.uint64)
    bo = np.concatenate([[0], np.cumsum(bl)[:-1]]).astype(np.uint64)
    rng = np.random.default_rng(3)
    cuts = np.unique(np.concatenate([[0, n], rng.integers(0, n, 700)])).astype(np.uint64)
    with eng.reader(didx) as r:
        st, got, bst = r.read(cuts[:-1], np.diff(cuts), (base, bo, bl, np.arange(len(blobs), dtype=np.uint64)), out="device")
        assert (bst == _lib.DEC_OK).all() and (st == _lib.DEC_OK).all()
        out = torch.cat(got)
        assert (eng.sha256_batch(out, [0], [n]) == eng.sha256_batch(data, [0], [n])).all()
        # the default cache holds 256 MiB: the first chunks were evicted by later groups, the last ones are cached
        need = r.plan([0, n - 1], [1, 1])[0].tolist()
        assert need == [0]


def test_blobs_of_untouched_chunks_are_cached(eng):
    didx, _, archive, store = write_snapshot(eng, [content(1_200_000, 600)], "lzh")
    ends, digs = eng.didx_parse(didx)
    starts = [0] + [int(x) for x in ends[:-1]]
    with eng.reader(didx) as r:
        st, data, bst = r.read([starts[1]], [10], {c: store[bytes(digs[c])] for c in (1, 4, 5)})
        assert st[0] == _lib.DEC_OK and (bst == _lib.DEC_OK).all()
        assert r.plan([starts[4], starts[5]], [5, 5])[0].tolist() == []
        st, data, _ = r.read([starts[4]], [int(ends[5]) - starts[4]], {})
        assert st[0] == _lib.DEC_OK and data[0] == archive[starts[4]:int(ends[5])]


# ---- 4. statuses ----------------------------------------------------------------------------------------------
def spans(ends):
    return [(0 if c == 0 else ends[c - 1], ends[c]) for c in range(len(ends))]


def test_every_status_between_intact_neighbours(eng):
    body = [content(n, 700 + i) for i, n in enumerate([30_000, 50_000, 40_000])]
    data = b"".join(transfer.payload_header(len(f)) + f for f in body)
    p1 = 16 + len(body[0])                       # payload offset of file 1
    # file 1's header straddles chunks 1 and 3; chunk 2 is empty; chunks 3 and 4 have one length (a blob of the other
    # decodes to the right size and fails on its digest)
    ends = [20_000, p1 + 8, p1 + 8, p1 + 30_008, p1 + 60_008, len(data)]
    didx, blobs = manual_archive(eng, data, ends)
    sp = spans(ends)
    with eng.crypt(KEY) as crypt:
        didx_e, blobs_e = manual_archive(eng, data, ends, "lzh", crypt)
        good = dict(enumerate(blobs))
        out = np.full(len(data), SENT, np.uint8)

        def check(r, blobs, ranges, want, flags=0):
            out[:] = SENT
            st, bst = raw_read(eng, r, [a for a, _ in ranges], [n for _, n in ranges], blobs, out, [a for a, _ in ranges], flags)
            assert st.tolist() == want, (st.tolist(), want)
            for (a, n), s in zip(ranges, st):
                hs = 16 if flags else 0
                if s == _lib.DEC_OK:
                    assert out[a:a + n].tobytes() == data[a + hs:a + hs + n]
            return bst

        def bad_bytes_absent(c, ranges, flags=0):
            """no byte of chunk c's span reached `out` (output offsets equal archive offsets in these checks)"""
            a, e = sp[c]
            hs = 16 if flags else 0
            for o, n in ranges:
                lo, hi = max(a - hs, o), min(e - hs, o + n)
                if lo < hi:
                    assert (out[lo:hi] == SENT).all(), (c, o, n)

        whole = lambda c: (sp[c][0], sp[c][1] - sp[c][0])
        across = (sp[3][0] + 100, sp[5][0] - sp[3][0])             # from inside chunk 3 to inside chunk 5
        with eng.reader(didx) as r:
            # missing: chunk 4 neither cached nor given
            check(r, {3: good[3], 5: good[5]}, [whole(3), across, whole(5)], [0, _lib.DEC_MISSING, 0])
            bad_bytes_absent(4, [across])
        with eng.reader(didx) as r:
            flip = bytearray(good[4]); flip[len(flip) // 2] ^= 0x10
            bst = check(r, {3: good[3], 4: bytes(flip), 5: good[5]}, [whole(3), across, whole(5)], [0, _lib.DEC_BAD_CRC, 0])
            assert bst.tolist() == [0, _lib.DEC_BAD_CRC, 0]
            bad_bytes_absent(4, [across])
            assert r.plan(*whole(4))[0].tolist() == [4]
            # another chunk's valid blob
            check(r, {4: good[3]}, [whole(3), across, whole(5)], [0, _lib.DEC_BAD_DIGEST, 0])
            bad_bytes_absent(4, [across])
            # a cached chunk given again with a corrupt blob: its status, and it leaves the cache
            check(r, {4: good[4]}, [across], [0])
            assert r.plan(*whole(4))[0].tolist() == []
            check(r, {4: bytes(flip)}, [whole(3), across, whole(5)], [0, _lib.DEC_BAD_CRC, 0])
            bad_bytes_absent(4, [across])
            assert r.plan(*whole(4))[0].tolist() == [4]
            # the PAYLOAD header: straddling chunks 1 and 3 (the empty chunk 2 between them is never touched), an
            # offset off by one, a wrong size
            check(r, good, [(p1, len(body[1])), (0, len(body[0])), (p1 + 16 + len(body[1]), len(body[2]))], [0, 0, 0],
                  _lib.READ_PAYLOAD)
            check(r, {}, [(p1 + 1, len(body[1]) - 1), (p1, len(body[1]) + 1), (0, len(body[0]))],
                  [_lib.DEC_BAD_HEADER, _lib.DEC_BAD_HEADER, 0], _lib.READ_PAYLOAD)
            assert r.plan([p1], [len(body[1])], payload=True)[0].tolist() == []
        with eng.reader(didx_e) as r:                 # encrypted blobs without a crypt
            enc = dict(enumerate(blobs_e))
            check(r, {3: enc[3], 4: enc[4], 5: enc[5]}, [whole(3)], [_lib.DEC_ENCRYPTED])
        with eng.reader(didx_e, crypt=crypt) as r:    # a forged tag
            forged = bytearray(blobs_e[4]); forged[30] ^= 1
            bst = check(r, {3: enc[3], 4: bytes(forged), 5: enc[5]}, [whole(3), across, whole(5)], [0, _lib.DEC_BAD_TAG, 0])
            assert bst.tolist() == [0, _lib.DEC_BAD_TAG, 0]
            bad_bytes_absent(4, [across])
            check(r, {4: enc[4]}, [across], [0])


# ---- 5. outputs and bases -------------------------------------------------------------------------------------
def test_host_and_device_outputs_and_blob_bases(eng, torch):
    didx, _, archive, store = write_snapshot(eng, [content(900_000, 800)], "lzl")
    ends, digs = eng.didx_parse(didx)
    n_chunks = len(ends)
    rng = np.random.default_rng(4)
    off = rng.integers(0, len(archive) - 70_000, 40).astype(np.uint64)
    ln = rng.integers(0, 70_000, 40).astype(np.uint64)
    oo = np.concatenate([[3], 3 + np.cumsum(ln + 5)[:-1]]).astype(np.uint64)   # ragged, with gaps
    total = int(oo[-1] + ln[-1]) + 16
    blobs = [store[bytes(digs[c])] for c in range(n_chunks)]
    pos = 7
    bo = []
    for b in blobs:
        bo.append(pos)
        pos += len(b) + 3
    dev_base = np.full(pos, 0xEE, np.uint8)
    for b, o in zip(blobs, bo):
        dev_base[o:o + len(b)] = np.frombuffer(b, np.uint8)
    dbase = torch.from_numpy(dev_base).cuda()
    bo = np.array(bo, np.uint64)
    bl = np.array([len(b) for b in blobs], np.uint64)
    for where in ("host", "device"):
        for src in ("host", "device"):
            with eng.reader(didx) as r:
                out = np.full(total, SENT, np.uint8) if where == "host" else torch.full((total,), SENT, dtype=torch.uint8, device="cuda")
                st = np.full(40, -1, np.int32)
                base = dev_base if src == "host" else dbase
                eng._ck(eng._L.pbsgpu_reader_read(r._h, off.ctypes.data, ln.ctypes.data, 40, 0, _ptr(base), bo.ctypes.data,
                                                  bl.ctypes.data, np.arange(n_chunks, dtype=np.uint64).ctypes.data, n_chunks,
                                                  _ptr(out), oo.ctypes.data, st.ctypes.data, None))
                assert (st == 0).all()
                h = out if where == "host" else out.cpu().numpy()
                for i in range(40):
                    a = int(off[i])
                    assert h[int(oo[i]):int(oo[i] + ln[i])].tobytes() == archive[a:a + int(ln[i])], (where, src, i)
                gaps = np.ones(total, bool)
                for i in range(40):
                    gaps[int(oo[i]):int(oo[i] + ln[i])] = False
                assert (h[gaps] == SENT).all()
            # the Python form with a device base
            with eng.reader(didx) as r:
                st, data, _ = r.read(off, ln, (dbase, bo, bl, np.arange(n_chunks)), out=where)
                assert (st == 0).all()
                got = data if where == "host" else [d.cpu().numpy().tobytes() for d in data]
                assert got == [archive[int(a):int(a + n)] for a, n in zip(off, ln)]


# ---- 6. lifecycle and arguments -------------------------------------------------------------------------------
def test_two_readers_are_independent_and_close_returns_the_cache(eng, torch):
    didx, _, archive, store = write_snapshot(eng, [content(300_000, 900)], "z")
    ends, digs = eng.didx_parse(didx)
    with eng.reader(didx) as r1, eng.reader(didx) as r2:
        st, _, _ = r1.read([0], [100], {0: store[bytes(digs[0])]})
        assert st[0] == 0 and len(r1.plan([0], [100])[0]) == 0
        assert r2.plan([0], [100])[0].tolist() == [0]
        assert r2.read([0], [100], {})[0][0] == _lib.DEC_MISSING
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    r = eng.reader(didx, cache_bytes=2 << 30)
    assert torch.cuda.mem_get_info()[0] <= free0 - (2 << 30)
    r.close()
    assert torch.cuda.mem_get_info()[0] >= free0 - (64 << 20)


def test_argument_errors(eng):
    didx, _, archive, store = write_snapshot(eng, [content(200_000, 1000)], "z")
    ends, digs = eng.didx_parse(didx)
    size = len(archive)
    L = eng._L
    with eng.reader(didx) as r:
        assert r.size == size
        for off, n, payload in [(size - 5, 6, False), (size + 1, 0, False), (size - 20, 5, True), (2**64 - 1, 2, False)]:
            with pytest.raises(pg.PbsGpuError) as e:
                r.plan([off], [n], payload)
            assert e.value.code == _lib.EINVAL
            with pytest.raises(pg.PbsGpuError) as e:
                r.read([off], [n], {}, payload)
            assert e.value.code == _lib.EINVAL
        b0 = store[bytes(digs[0])]
        for bad in [(b"".join([b0, b0]), [0, len(b0)], [len(b0)] * 2, [0, 0]), (b0, [0], [len(b0)], [len(ends)])]:
            with pytest.raises(pg.PbsGpuError) as e:
                r.read([0], [10], (np.frombuffer(bad[0], np.uint8), bad[1], bad[2], bad[3]))
            assert e.value.code == _lib.EINVAL
        o = np.zeros(1, np.uint64)
        l = np.ones(1, np.uint64)
        st = np.zeros(1, np.int32)
        out = np.zeros(16, np.uint8)
        n = C.c_uint64()
        assert L.pbsgpu_reader_read(r._h, None, l.ctypes.data, 1, 0, None, None, None, None, 0, out.ctypes.data, o.ctypes.data,
                                    st.ctypes.data, None) == _lib.EINVAL
        assert L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, 1, 0, None, None, None, None, 0, None, o.ctypes.data,
                                    st.ctypes.data, None) == _lib.EINVAL
        assert L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, 1, 0, None, None, None, None, 1, out.ctypes.data,
                                    o.ctypes.data, st.ctypes.data, None) == _lib.EINVAL
        assert L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, 1, 2, None, None, None, None, 0, out.ctypes.data,
                                    o.ctypes.data, st.ctypes.data, None) == _lib.EINVAL
        assert L.pbsgpu_reader_plan(r._h, o.ctypes.data, l.ctypes.data, 1, 0, None, None, 0, None) == _lib.EINVAL
        assert L.pbsgpu_reader_plan(r._h, o.ctypes.data, l.ctypes.data, 1, 0, None, None, 0, C.byref(n)) == _lib.ERANGE
        assert n.value == 1
        # a range that ends exactly at the end is fine; a zero-length plain range touches nothing
        assert r.plan([size - 5], [5])[0].tolist() == [len(ends) - 1]
        st, data, _ = r.read([7], [0], {})
        assert st[0] == 0 and data == [b""]
    with pg.Engine(0) as other, other.crypt(KEY) as foreign:
        with pytest.raises(pg.PbsGpuError) as e:
            eng.reader(didx, crypt=foreign)
        assert e.value.code == _lib.EINVAL
    bad = bytearray(didx); bad[40] ^= 1                     # index_csum
    with pytest.raises(pg.PbsGpuError) as e:
        eng.reader(bytes(bad))
    assert e.value.code == _lib.EINVAL
    dec = bytearray(didx)                                    # decreasing ends (csum fixed up)
    dec[4096:4104] = (int(ends[1]) + 1).to_bytes(8, "little")
    dec[32:64] = hashlib.sha256(bytes(dec[4096:])).digest()
    with pytest.raises(pg.PbsGpuError) as e:
        eng.reader(bytes(dec))
    assert e.value.code == _lib.EINVAL
