"""Fixed indexes (.fidx) on the GPU: fixed cuts through the batch job (host and device bases, several streams at every
offset residue mod 16, the async form with and without early input release), set flags, keyed digests, slices, the
index round trip and seeding, and the archive reader over a .fidx with blobs of every encoder, plain and encrypted."""
import ctypes as C
import hashlib
import os
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

import crypt_ref
import fidx_ref
import pbs_plus_b200 as pg
import zstd_lz_ref as lzref
from pbs_plus_b200 import _lib, transfer

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
KEY = bytes(range(11, 43))
IDENT = crypt_ref.id_key(KEY)
K = 5
TEXT = lzref.text_corpus(1 << 20, 1)


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


def image(n: int, seed: int) -> bytes:
    """4 KiB blocks of text, zeros and random bytes: compressible and raw blocks, and repeated (zero) chunks."""
    rng = np.random.default_rng(seed)
    blocks = max(1, -(-n // 4096))
    out = np.empty(blocks * 4096, np.uint8)
    for k, p in enumerate(rng.integers(0, 3, blocks)):
        at = (seed * 4096 + k * 4096) % (len(TEXT) - 4096)
        out[k * 4096:(k + 1) * 4096] = (TEXT[at:at + 4096] if p == 0 else
                                        np.zeros(4096, np.uint8) if p == 1 else rng.integers(0, 256, 4096, dtype=np.uint8))
    return out[:n].tobytes()


def lengths(cs: int) -> list[int]:
    return [0, 1, cs - 1, cs, cs + 1, K * cs, K * cs + 17]


def expected(streams: list[bytes], cs: int, key: bytes | None = None, seen: set | None = None) -> np.ndarray:
    """Records of a fixed-cut batch: (stream, end_off) order, digests from hashlib; with `seen` the set's flags."""
    rows = []
    for s, data in enumerate(streams):
        for i, d in enumerate(fidx_ref.chunk_digests(data, cs, key)):
            flags = 0
            if seen is not None:
                flags = int(d in seen)
                seen.add(d)
            rows.append((s, flags, min((i + 1) * cs, len(data)), np.frombuffer(d, np.uint8)))
    return np.array(rows, dtype=_lib.CHUNK_DTYPE)


def pack(streams: list[bytes]):
    """Stream i at an offset of residue i mod 16 -> (host buffer, off, len)."""
    off, pos = [], 0
    for i, s in enumerate(streams):
        pos = (pos + 255) // 256 * 256 + i % 16
        off.append(pos)
        pos += len(s)
    buf = np.zeros(pos + 1, np.uint8)
    for o, s in zip(off, streams):
        buf[o:o + len(s)] = np.frombuffer(s, np.uint8)
    return buf, np.array(off, np.uint64), np.array([len(s) for s in streams], np.uint64)


def streams_for(cs: int, seed: int) -> list[bytes]:
    ls = lengths(cs)
    return [image(ls[i % len(ls)], seed + i) for i in range(16)]


@pytest.mark.parametrize("cs", [4 << 10, 64 << 10, 4 << 20])
def test_records_match_hashlib_from_host_and_device(eng, torch, cs):
    streams = streams_for(cs, cs)
    buf, off, ln = pack(streams)
    want = expected(streams, cs)
    got = eng.chunk_digest_batch(None, buf, off, ln, fixed_size=cs)
    assert got.tobytes() == want.tobytes()
    dev = torch.from_numpy(buf).cuda()
    assert eng.chunk_digest_batch(None, dev, off, ln, fixed_size=cs).tobytes() == want.tobytes()
    for early in (False, True):
        job = eng.submit(None, dev, off, ln, early_input=early, fixed_size=cs)
        job.wait_input()
        rec, t = job.wait()
        assert rec.tobytes() == want.tobytes(), early
        assert t["scan_launches"] == 0 and t["candidates"] == 0 and t["reruns"] == 0
    # one stream per call, every length of the table alone
    for s in streams[:7]:
        b, o, l = pack([s])
        assert eng.chunk_digest_batch(None, b, o, l, fixed_size=cs).tobytes() == expected([s], cs).tobytes()


def test_set_flags_equal_a_python_walk(eng, torch):
    cs = 4 << 10
    streams = [image(40 * cs + 5, 1), bytes(9 * cs), image(3 * cs, 1)[: 3 * cs], bytes(cs + 3)]   # zero chunks repeat
    buf, off, ln = pack(streams)
    seen: set = set()
    known = eng.digest_set()
    first = eng.chunk_digest_batch(None, buf, off, ln, known, fixed_size=cs)
    assert first.tobytes() == expected(streams, cs, seen=seen).tobytes()
    assert first["flags"].sum() > 8                                                 # repeated zero chunks within the call
    more = [image(7 * cs + 1, 2), bytes(2 * cs)]
    b2, o2, l2 = pack(more)
    job = eng.submit(None, torch.from_numpy(b2).cuda(), o2, l2, known, fixed_size=cs)
    rec, _ = job.wait()
    assert rec.tobytes() == expected(more, cs, seen=seen).tobytes()
    assert len(known) == len(seen)


def test_keyed_digests_equal_the_restatement(eng, torch):
    cs = 64 << 10
    streams = streams_for(cs, 7)
    buf, off, ln = pack(streams)
    with eng.crypt(KEY) as crypt:
        seen: set = set()
        known = eng.digest_set()
        got = eng.chunk_digest_batch(None, buf, off, ln, known, crypt=crypt, fixed_size=cs)
        assert got.tobytes() == expected(streams, cs, IDENT, seen).tobytes()
        rec, _ = eng.submit(None, torch.from_numpy(buf).cuda(), off, ln, crypt=crypt, fixed_size=cs).wait()
        assert rec.tobytes() == expected(streams, cs, IDENT).tobytes()


def test_batch_opts_sizes_and_argument_errors(eng):
    cfg = pg.make_config(1 << 12)
    data = image(300_000, 3)
    buf, off, ln = pack([data])
    out = np.zeros(4096, dtype=_lib.CHUNK_DTYPE)
    n = C.c_uint64()

    def call(size, fixed, cfg_ref, n_forced=0):
        o = _lib.BatchOptsFixed()
        o.size, o.fixed_size = size, fixed
        fs, fo = np.zeros(1, np.uint32), np.array([1000], np.uint64)
        if n_forced:
            o.forced_stream, o.forced_off, o.n_forced = fs.ctypes.data, fo.ctypes.data, 1
        rc = eng._L.pbsgpu_chunk_digest_batch_ex(eng._h, cfg_ref, buf.ctypes.data, off.ctypes.data, ln.ctypes.data, 1,
                                                 C.byref(o), out.ctypes.data, len(out), C.byref(n))
        return rc, out[: n.value].copy()

    chunker = eng.chunk_digest_batch(cfg, buf, off, ln)
    for old in (48, 56):                                  # the layouts without fixed_size: the chunker, field ignored
        rc, rec = call(old, 4096, C.byref(cfg))
        assert rc == 0 and rec.tobytes() == chunker.tobytes(), old
    rc, rec = call(64, 4096, None)
    assert rc == 0 and rec.tobytes() == expected([data], 4096).tobytes()
    rc, rec = call(64, 0, C.byref(cfg))
    assert rc == 0 and rec.tobytes() == chunker.tobytes()
    for bad in (2048, 4097, 3 * 4096, 32 << 20, 1 << 31):
        assert call(64, bad, None)[0] == _lib.EINVAL, bad
    assert call(64, 4096, None, n_forced=1)[0] == _lib.EINVAL
    assert call(64, 0, None)[0] == _lib.EINVAL            # the chunker still needs its cfg
    assert call(60, 4096, None)[0] == _lib.EINVAL


def test_slices_give_the_digests_of_one_call(eng, torch):
    cs = 64 << 10
    data = image(37 * cs + 123, 4)
    whole = eng.chunk_digest_batch(None, np.frombuffer(data, np.uint8), [0], [len(data)], fixed_size=cs)
    for step, dev in ((cs, False), (8 * cs, True), (len(data), False)):
        w = transfer.FixedIndexWriter(eng, cs)
        for a in range(0, len(data), step):
            part = np.frombuffer(data[a:a + step], np.uint8)
            w.WriteSlice(torch.from_numpy(part.copy()).cuda() if dev else part)
        assert w.size == len(data) and w.digests == [bytes(d) for d in whole["digest"]], step
        assert w.fidx(bytes(range(16)), 99) == fidx_ref.fidx_build(w.digests, len(data), cs, bytes(range(16)), 99)
    w = transfer.FixedIndexWriter(eng, cs)
    w.WriteSlice(data[:cs + 1])
    with pytest.raises(ValueError):
        w.WriteSlice(data[cs + 1:])                        # a slice after one that ended inside a chunk


def test_index_round_trip_verify_and_seed(eng):
    cs = 4 << 10
    for size in (0, 1, cs, 123 * cs + 17):
        data = image(size, 5)
        dig = fidx_ref.chunk_digests(data, cs)
        img = eng.fidx_build(b"".join(dig), size, cs, bytes(range(16)), -7)
        assert img == fidx_ref.fidx_build(dig, size, cs, bytes(range(16)), -7)
        s, c, d = eng.fidx_parse(img)
        assert (s, c) == (size, cs) and [bytes(x) for x in d] == dig
    with pytest.raises(pg.PbsGpuError):
        eng.fidx_build(b"".join(dig[:-1]), size, cs)         # one digest short
    bad = bytearray(img)
    bad[4096 + 32 * 5 + 3] ^= 1
    assert eng.fidx_parse(bytes(bad), verify=False)[0] == size
    with pytest.raises(pg.PbsGpuError) as e:
        eng.fidx_parse(bytes(bad))
    assert e.value.code == _lib.EINVAL
    with pytest.raises(pg.PbsGpuError):
        eng.reader_fidx(bytes(bad))                         # the reader verifies the checksum too
    known = eng.digest_set()
    assert known.seed_fidx(img) == len(dig)
    rec = eng.chunk_digest_batch(None, np.frombuffer(data, np.uint8), [0], [size], known, fixed_size=cs)
    assert len(rec) == len(dig) and (rec["flags"] == 1).all()
    with pytest.raises(pg.PbsGpuError):
        known.seed_fidx(img[:-1])


def write_image(eng, data: bytes, cs: int, mode: str, key: bytes | None):
    store = {}
    w = transfer.FixedIndexWriter(eng, cs, eng.digest_set(), upload_blob=store.__setitem__, blob_compression=mode,
                                  crypt_key=key)
    w.WriteSlice(data)
    return w.fidx(), store


def random_ranges(size: int, n: int, seed: int, cs: int):
    rng = random.Random(seed)
    out = [(0, size), (0, 0), (size, 0), (max(0, size - 1), min(1, size))]
    for _ in range(n):
        a = rng.randrange(0, size + 1)
        out.append((a, rng.randrange(0, min(size - a, 3 * cs) + 1)))
    return out


@pytest.mark.parametrize("mode,key", [("z", None), ("lz", None), ("lze", None), ("lzh", None), ("lzl", None),
                                      ("lzh", KEY), ("raw", KEY)])
def test_reader_over_fidx(eng, mode, key):
    cs = 64 << 10
    data = image(29 * cs + 4321, 6)
    if mode == "raw":                                     # uncompressed blobs: FixedIndexWriter writes compressed modes
        a = np.frombuffer(data, np.uint8)
        off = np.arange(0, len(data), cs, dtype=np.uint64)
        ln = np.minimum(np.uint64(len(data)) - off, np.uint64(cs))
        crypt = eng.crypt(key)
        dig = eng.sha256_keyed_batch(crypt, a, off, ln)
        blobs = eng.blob_encode_batch_enc(crypt, "raw", a, off, ln, os.urandom(16 * len(off)))[0]
        crypt.close()
        fidx = eng.fidx_build(dig, len(data), cs)
        store = {bytes(d): b for d, b in zip(dig, blobs)}
    else:
        fidx, store = write_image(eng, data, cs, mode, key)
    crypt = eng.crypt(key) if key else None
    with eng.reader_fidx(fidx, crypt, cache_bytes=8 * cs) as r:
        assert r.size == len(data)
        for i, (o, l) in enumerate(random_ranges(len(data), 40, hash(mode) & 0xFFFF, cs)):
            chunks, dig = r.plan([o], [l])
            blobs = {int(c): store[bytes(d)] for c, d in zip(chunks, dig)}
            st, got, bst = r.read([o], [l], blobs)
            assert st.tolist() == [0] and (bst == 0).all() and got[0] == data[o:o + l], (i, o, l)
        with pytest.raises(pg.PbsGpuError) as e:
            r.plan([0], [10], payload=True)
        assert e.value.code == _lib.EINVAL
        with pytest.raises(pg.PbsGpuError):
            r.read([0], [len(data) + 1], {})
    if crypt is not None:
        crypt.close()


def test_reader_over_fidx_corrupt_blob_sets_only_its_status(eng, torch):
    cs = 4 << 10
    data = image(50 * cs + 9, 8)
    fidx, store = write_image(eng, data, cs, "lzh", None)
    _, _, dig = eng.fidx_parse(fidx)
    with eng.reader_fidx(fidx) as r:
        blobs = {c: store[bytes(dig[c])] for c in range(len(dig))}
        bad = bytearray(blobs[7]); bad[-1] ^= 0x40; blobs[7] = bytes(bad)
        ranges = [(0, 7 * cs), (6 * cs + 5, 2 * cs), (7 * cs, 1), (8 * cs, len(data) - 8 * cs)]
        for out in ("host", "device"):
            st, got, bst = r.read([a for a, _ in ranges], [b for _, b in ranges], blobs, out=out)
            assert st.tolist() == [0, _lib.DEC_BAD_CRC, _lib.DEC_BAD_CRC, 0]
            assert bst.tolist() == [_lib.DEC_BAD_CRC if c == 7 else 0 for c in range(len(dig))]
            for k in (0, 3):
                a, b = ranges[k]
                g = got[k] if out == "host" else got[k].cpu().numpy().tobytes()
                assert g == data[a:a + b]
            r.read([0], [0], {}, out=out)


def test_cxx_fixed_index_writer(eng, tmp_path):
    """include/pbsgpu.hpp's FixedIndexWriter (tests/cxx/fidx_driver.cpp): digests, flags, blobs and the .fidx."""
    drv = ROOT / "tests" / "cxx" / "fidx_driver.bin"
    cs = 64 << 10
    data = image(21 * cs + 5, 9) + bytes(3 * cs)
    f = tmp_path / "disk.img"
    f.write_bytes(data)
    out = subprocess.run([str(drv), str(cs), str(f), str(tmp_path / "disk.img.fidx")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.split("\n")
    dig = fidx_ref.chunk_digests(data, cs)
    seen: set = set()
    want = []
    for d in dig:
        want.append(f"chunk {d.hex()} {int(d in seen)}")
        seen.add(d)
    assert [x for x in lines if x.startswith("chunk ")] == want
    blobs = [x.split() for x in lines if x.startswith("blob ")]
    first = {}
    for i, d in enumerate(dig):
        first.setdefault(d, min(cs, len(data) - i * cs))
    assert [(b[1], int(b[2])) for b in blobs] == [(d.hex(), n) for d, n in first.items()]
    st, _, _ = eng.blob_decode_batch([bytes.fromhex(b[3]) for b in blobs], [int(b[2]) for b in blobs],
                                     b"".join(bytes.fromhex(b[1]) for b in blobs), out=None)
    assert (st == 0).all()
    assert (tmp_path / "disk.img.fidx").read_bytes() == fidx_ref.fidx_build(dig, len(data), cs)
    assert "seeded-rerun-known all" in lines
