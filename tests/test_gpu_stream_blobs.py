"""DataBlobs of new chunks and XXH3-64 of byte ranges from the streaming form (pbsgpu_stream_blob_mode / _poll_blobs,
pbsgpu_stream_hash_range / _poll_hashes) and the payload-stream writer built on them."""
import ctypes as C
import io
import os
import zlib

import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg
import zstd_ent_ref as entref
import zstd_lz_ref as lzref
from oracle import pyref
from pbs_plus_b200 import transfer
from pbs_plus_b200._lib import CHUNK_KNOWN, EINVAL, ESTATE
from test_gpu_round2 import _payload_stream, rnd
from test_gpu_zstd_lz import decode

pytestmark = pytest.mark.gpu
MODES = ["raw", "z", "lz", "lze"]


def engine(window):
    old = os.environ.get("PBSGPU_STREAM_WINDOW")
    os.environ["PBSGPU_STREAM_WINDOW"] = str(window)
    try:
        return pg.Engine(0)
    finally:
        if old is None:
            del os.environ["PBSGPU_STREAM_WINDOW"]
        else:
            os.environ["PBSGPU_STREAM_WINDOW"] = old


@pytest.fixture(scope="module")
def eng1m():
    e = engine(1 << 20)
    yield e
    e.close()


def batch_blobs(e, mode, data, off, ln):
    if mode == "raw":
        out, boff, _ = e.blob_encode_batch(data, off, ln)
        return [out[int(boff[i]): int(boff[i + 1])].tobytes() for i in range(len(off))]
    return getattr(e, "blob_encode_batch_" + mode)(data, off, ln)[0]


def mixed_files():
    text = lzref.text_corpus(700_000, seed=7)
    rep = rnd(300_000, 11)
    return [text, np.zeros(400_000, np.uint8), rnd(250_001, 12), rep, lzref.text_corpus(333_333, seed=8), rep,
            rnd(5, 13), np.zeros(1, np.uint8), rnd(180_000, 14)]


def write_stream(st, files, split, poll_each):
    """The payload stream of `files` written in pieces of `split` bytes, a suggested boundary at every file start."""
    rec, blobs = [], []
    st.write(np.frombuffer(transfer.PXAR_PAYLOAD_START_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little"), np.uint8))
    for f in files:
        st.suggest(st.position)
        data = np.concatenate([np.frombuffer(transfer.payload_header(len(f)), np.uint8), f])
        for p in range(0, len(data), split):
            st.write(data[p: p + split])
            if poll_each:
                rec.append(st.poll(1 << 16))
                blobs += st.poll_blobs()
    st.write(np.frombuffer(transfer.PXAR_PAYLOAD_TAIL_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little"), np.uint8))
    rec.append(st.finish())
    blobs += st.poll_blobs()
    return np.concatenate(rec), blobs


@pytest.mark.parametrize("mode", MODES)
def test_stream_blobs_equal_the_batch_encoders(eng1m, mode):
    e = eng1m
    files = mixed_files()
    stream, starts = _payload_stream(files)
    avg = 1 << 16
    ref = oracle.chunk_digest_forced(oracle.config(avg), stream, np.array(starts, np.uint64))
    ends = ref["end_off"].astype(np.uint64)
    seeded = ref["digest"][(ref["end_off"] > starts[2]) & (ref["end_off"] <= starts[3])]   # the random file's chunks
    assert len(seeded) >= 2
    oset = oracle.DigestSet()
    oset.probe(seeded, insert=True)
    known = oset.probe(ref["digest"], insert=True).astype(bool)
    off = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    ln = ends - off
    want = batch_blobs(e, mode, stream, off[~known], ln[~known])
    got = []
    for split, poll_each in ((100_003, True), (77_777, False)):
        ds = e.digest_set()
        ds.insert(seeded)
        st = e.stream(pg.make_config(avg), ds)
        st.blob_mode(mode)
        rec, blobs = write_stream(st, files, split, poll_each)
        st.close()
        assert rec["end_off"].tolist() == ref["end_off"].tolist() and rec["digest"].tobytes() == ref["digest"].tobytes()
        assert ((rec["flags"] & CHUNK_KNOWN) != 0).tolist() == known.tolist()
        assert len(blobs) == int((~known).sum()) and blobs == want
        got.append(blobs)
    assert got[0] == got[1]
    chunks = [stream[int(o): int(o + l)].tobytes() for o, l in zip(off[~known], ln[~known])]
    if mode in ("lz", "lze"):
        restate = lzref.blob_encode_lz if mode == "lz" else entref.blob_encode_lze
        for b, c in list(zip(got[0], chunks))[::3]:
            assert b == restate(c)
    for b, c in list(zip(got[0], chunks))[::4]:
        if b[:8] == pyref.BLOB_MAGIC_COMPRESSED:
            assert decode(b[12:], len(c)) == c
        else:
            assert b[12:] == c


def test_payload_writer_uploads_blobs_of_new_chunks_only(eng1m):
    e = eng1m
    avg = 1 << 14
    files = [rnd(n, 40 + i) for i, n in enumerate([400_000, 300_000, 500_000])]
    w0 = transfer.PayloadStreamWriter(e, pg.make_config(avg))
    offs = [w0.WriteEntryReader(transfer.Entry(f"f{i}", len(f)), io.BytesIO(f.tobytes()), len(f)) for i, f in enumerate(files)]
    w0.Finish()
    image = w0.didx()
    ends, digs = e.didx_parse(image)
    known = e.digest_set()
    known.seed_didx(image)
    up = []
    w1 = transfer.PayloadStreamWriter(e, pg.make_config(avg), known, prev_index=(ends, digs),
                                      upload_blob=lambda d, b: up.append((d, b)), blob_compression="lze",
                                      hash_files=True)
    new = np.concatenate([lzref.text_corpus(200_000, seed=3), rnd(250_000, 99)])
    w1.WriteEntryReader(transfer.Entry("new", len(new)), io.BytesIO(new.tobytes()), len(new))
    w1.WriteEntryRef(transfer.Entry("f1", len(files[1])), offs[1])
    w1.WriteEntryReader(transfer.Entry("f0b", len(files[0])), io.BytesIO(files[0].tobytes()), len(files[0]))
    w1.WriteEntryReader(transfer.Entry("new2", 70_000), io.BytesIO(new[:70_000].tobytes()), 70_000)
    w1.Finish()
    # the oracle: the two pbsgpu streams the writer chunked (before and after the injected chunks)
    marker = lambda m: np.frombuffer(m.to_bytes(8, "little") + (16).to_bytes(8, "little"), np.uint8)
    hdr = lambda f: np.frombuffer(transfer.payload_header(len(f)), np.uint8)
    seg1 = np.concatenate([marker(transfer.PXAR_PAYLOAD_START_MARKER), hdr(new), new])
    seg2 = np.concatenate([hdr(files[0]), files[0], hdr(new[:70_000]), new[:70_000], marker(transfer.PXAR_PAYLOAD_TAIL_MARKER)])
    oset = oracle.DigestSet()
    oset.probe(digs, insert=True)
    want = []
    for seg, starts in ((seg1, [16]), (seg2, [16 + len(files[0])])):
        ref = oracle.chunk_digest_forced(oracle.config(avg), seg, np.array(starts, np.uint64))
        k = oset.probe(ref["digest"], insert=True).astype(bool)
        end = ref["end_off"].astype(np.uint64)
        off = np.concatenate([[0], end[:-1]]).astype(np.uint64)
        blobs = e.blob_encode_batch_lze(seg, off[~k], (end - off)[~k])[0]
        want += list(zip([bytes(d) for d in ref["digest"][~k]], blobs))
    assert up == want
    old = {bytes(d) for d in digs}
    assert not any(d in old for d, _ in up)
    assert len({d for d, _ in up}) == len(up)
    assert [x[1] for x in w1.index if not x[2]] == [d for d, _ in up]
    assert set(w1.backed_hashes) == {"new", "f0b", "new2"}
    with pytest.raises(ValueError):
        transfer.PayloadStreamWriter(e, pg.make_config(avg), blob_compression="zz")


HASH_SIZES = [0, 1, 3, 4, 8, 9, 16, 17, 128, 129, 240, 241, 1023, 1024, 1025, 2048, 2049, 65535, 65536, 65537]


@pytest.mark.parametrize("window", [1 << 16, 3 << 16, 1 << 20])
def test_payload_writer_backed_hashes(window, tmp_path):
    """Every size class, at windows small enough that ranges cross window ends inside a block, inside the tail and
    inside a short range (several files, several windows' worth, written in odd reads)."""
    e = engine(window)
    try:
        sizes = HASH_SIZES + [5 * window + 12_345, 2 * window] + HASH_SIZES[::-1] + [700, 1100, 1500] * 30
        files = {f"d/f{i}": (lzref.text_corpus(n, seed=i) if i % 3 == 0 else rnd(n, 500 + i)) for i, n in enumerate(sizes)}
        for avg in (1 << 12, 1 << 14):
            w = transfer.PayloadStreamWriter(e, pg.make_config(avg), e.digest_set(), hash_files=True)
            for p, f in files.items():
                w.WriteEntryReader(transfer.Entry(p, len(f)), io.BufferedReader(io.BytesIO(f.tobytes()), 4099), len(f))
            w.Finish()
            assert set(w.backed_hashes) == set(files)
            want = {p: oracle.xxh3_64(f) for p, f in files.items()}
            assert w.backed_hashes == want, avg
        arrs = list(files.values())
        lens = np.array([len(a) for a in arrs], np.uint64)
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
        buf = np.concatenate(arrs) if arrs else np.zeros(1, np.uint8)
        assert e.xxh3_batch(buf, offs, lens).tolist() == [want[p] for p in files]
        for p, f in files.items():
            (tmp_path / p).parent.mkdir(exist_ok=True)
            (tmp_path / p).write_bytes(f.tobytes())
        opener = lambda rel: open(tmp_path / rel, "rb")
        transfer.verifyBackedFileHashes(e, opener, w.backed_hashes)
        raw = bytearray(files["d/f20"].tobytes())
        raw[len(raw) // 2] ^= 1
        (tmp_path / "d/f20").write_bytes(bytes(raw))
        with pytest.raises(IOError, match='backed file "d/f20" content hash differs'):
            transfer.verifyBackedFileHashes(e, opener, w.backed_hashes)
    finally:
        e.close()


def test_stream_hash_ranges_polled_as_they_finish(eng1m):
    """Direct use of the stream: ranges anywhere in the stream (not only file contents), polled after every write."""
    e = eng1m
    data = rnd(5_000_000, 77)
    st = e.stream(pg.make_config(1 << 16))
    rng = np.random.default_rng(5)
    ranges, pos = [], 0
    while True:
        o = pos + int(rng.integers(0, 3000))
        n = int(rng.choice([0, 1, 17, 240, 241, 1024, 1025, 4000, 70_000, 1_500_000]))
        if o + n > len(data):
            break
        ranges.append((o, n))
        pos = o + n
    got, k = [], 0
    for p in range(0, len(data), 65_521):
        while k < len(ranges) and ranges[k][0] >= st.position and ranges[k][0] < p + 65_521:
            st.hash_range(*ranges[k])
            k += 1
        st.write(data[p: p + 65_521])
        got += st.poll_hashes().tolist()
    st.finish()
    got += st.poll_hashes().tolist()
    st.close()
    assert k == len(ranges) and got == [oracle.xxh3_64(data[o: o + n]) for o, n in ranges]


def test_large_stream_reuses_windows(tmp_path):
    """6 GiB at the default 2 GiB windows (the buffers are reused): blobs counted, sampled blobs decode, all hashes."""
    e = pg.Engine(0)
    try:
        up, n_new = [], 0
        def keep(d, b):
            nonlocal n_new
            if n_new % 97 == 0:
                up.append((d, b))
            n_new += 1
        ds = e.digest_set(1 << 20)
        w = transfer.PayloadStreamWriter(e, pg.make_config(1 << 22), ds, upload_blob=keep, blob_compression="z",
                                         hash_files=True)
        base = rnd(96 << 20, 4242)
        f = np.zeros(128 << 20, np.uint8)
        want = {}
        for i in range(49):
            np.bitwise_xor(base, np.uint8(i), out=f[: 96 << 20])     # 96 MiB distinct per file, 32 MiB of zeros
            n = len(f) - i
            want[f"f{i}"] = int(e.xxh3_batch(f, [0], [n])[0])
            w.WriteEntryReader(transfer.Entry(f"f{i}", n), io.BytesIO(f[:n].tobytes()), n)
        idx = w.Finish()
        assert idx[-1][0] >= 6 << 30
        assert n_new == sum(1 for x in idx if not x[2]) and n_new > 1000   # one blob per record without KNOWN
        assert w.backed_hashes == want
        size = {x[1]: x[0] - (idx[k - 1][0] if k else 0) for k, x in enumerate(idx)}
        assert len(up) > 10
        for d, b in up:
            assert int.from_bytes(b[8:12], "little") == zlib.crc32(b[12:])
            if b[:8] == pyref.BLOB_MAGIC_COMPRESSED:
                assert len(decode(b[12:], size[d])) == size[d]
            else:
                assert len(b) == 12 + size[d]
    finally:
        e.close()


def test_stream_blob_and_hash_error_paths(eng1m):
    e = eng1m
    L = e._L
    st = e.stream(pg.make_config(1 << 16))
    assert L.pbsgpu_stream_blob_mode(st._h, 9) == EINVAL
    assert L.pbsgpu_stream_blob_mode(st._h, -1) == EINVAL
    st.hash_range(100, 50)
    assert L.pbsgpu_stream_hash_range(st._h, 120, 10) == EINVAL        # overlaps
    assert L.pbsgpu_stream_hash_range(st._h, 90, 5) == EINVAL          # not ascending
    st.write(rnd(1000, 1))
    assert L.pbsgpu_stream_blob_mode(st._h, 2) == ESTATE                # after the first byte
    assert L.pbsgpu_stream_hash_range(st._h, 500, 10) == EINVAL        # behind the write position
    n = C.c_uint64()
    small = np.zeros(1000, np.uint8)
    lens = np.zeros(4, np.uint64)
    assert L.pbsgpu_stream_poll_blobs(st._h, small.ctypes.data, len(small), lens.ctypes.data, 4, C.byref(n)) == EINVAL
    st.hash_range(2000, 10)                                             # past the end at finish
    with pytest.raises(pg.PbsGpuError):
        st.finish()
    st.close()
    out = np.zeros(4, np.uint64)
    assert L.pbsgpu_stream_blob_mode(None, 1) == EINVAL
    assert L.pbsgpu_stream_hash_range(None, 0, 1) == EINVAL
    assert L.pbsgpu_stream_poll_hashes(None, out.ctypes.data, 4, C.byref(n)) == EINVAL
    assert L.pbsgpu_stream_poll_blobs(None, small.ctypes.data, len(small), lens.ctypes.data, 4, C.byref(n)) == EINVAL
    with pytest.raises(ValueError):
        e.stream(pg.make_config(1 << 16)).blob_mode("zstd")


def _poll_window(st, timeout=30.0):
    """Records of the next collected window (its records arrive together)."""
    import time
    t0 = time.monotonic()
    while time.monotonic() - t0 < timeout:
        rec = st.poll(1 << 16)
        if len(rec):
            return rec
        time.sleep(0.001)
    raise AssertionError("no window was collected")


def test_stream_hash_ranges_cross_known_window_ends():
    """Without suggested boundaries a window of W bytes is consumed up to its last cut, so the window ends are known
    from the oracle's cuts: c_k = last cut <= c_(k-1) + W.  Ranges are placed so that each kind of span provably
    crosses one of them -- a 1 KiB block, a tail after the last block, a tail that overlaps the last block, a short
    range of each formula -- and a long range crosses two.  Every window end is checked against the records.  An
    empty range is registered and polled first, before any window is processed."""
    W, avg = 1 << 16, 4096
    e = engine(W)
    try:
        data = rnd(12 * W, 2024)
        cuts = oracle.chunk_digest(oracle.config(avg), data)["end_off"].astype(np.int64)
        ends, c = [], 0
        for _ in range(10):
            c = int(cuts[cuts <= c + W].max())
            ends.append(c)
        c1, c2, c3, c4, c5, c6, c7, c8 = ends[:8]
        ranges = [(50, 100),
                  (c1 - 5000, 10_000),     # block 4 of 9 crosses c1
                  (c2 - 3300, 3572),       # 3 blocks before c2, the tail crosses it
                  (c3 - 300, 700),         # short range (700 bytes: the 241..1024 formula) crosses c3
                  (c4 - 2060, 2078),       # 2 blocks before c4, the tail (which overlaps block 1) crosses it
                  (c5 - 50, 100),          # short range (<= 128 bytes) crosses c5
                  (c6 - 777, c8 + 999 - (c6 - 777))]   # blocks cross c6, c7 and c8
        assert (c1 - ranges[1][0]) % 1024 and ranges[2][0] + 3072 <= c2 < ranges[2][0] + 3572
        assert ranges[4][0] + 2048 <= c4 and ranges[4][0] + 2078 - 64 < c4 < ranges[4][0] + 2078
        st = e.stream(pg.make_config(avg))
        st.hash_range(0, 0)
        got = st.poll_hashes().tolist()
        assert got == [oracle.xxh3_64(data[:0])]
        for o, n in ranges:
            st.hash_range(o, n)
        pos, prev = 0, 0
        for k in range(8):
            st.write(data[pos: prev + W])
            pos = prev + W
            rec = _poll_window(st)
            assert int(rec["end_off"][-1]) == ends[k], k
            prev = ends[k]
            got += st.poll_hashes().tolist()
        st.write(data[pos:])
        st.finish()
        got += st.poll_hashes().tolist()
        st.close()
        assert got == [oracle.xxh3_64(data[:0])] + [oracle.xxh3_64(data[o: o + n]) for o, n in ranges]
    finally:
        e.close()


def test_payload_writer_hashes_more_files_than_one_poll_returns():
    """More than 65536 file ranges finish in one window (the last one, at Finish): every hash is drained."""
    e = engine(1 << 26)
    try:
        rng = np.random.default_rng(7)
        src = rnd(1 << 20, 8)
        sizes = rng.integers(0, 300, size=70_000)
        starts = rng.integers(0, len(src) - 300, size=len(sizes))
        w = transfer.PayloadStreamWriter(e, pg.make_config(1 << 12), e.digest_set(), hash_files=True)
        for i, (o, n) in enumerate(zip(starts.tolist(), sizes.tolist())):
            w.WriteEntryReader(transfer.Entry(f"f{i}", n), io.BytesIO(src[o: o + n].tobytes()), n)
        w.Finish()
        assert len(w.backed_hashes) == len(sizes)
        want = {f"f{i}": oracle.xxh3_64(src[o: o + n]) for i, (o, n) in enumerate(zip(starts.tolist(), sizes.tolist()))}
        assert w.backed_hashes == want
    finally:
        e.close()
