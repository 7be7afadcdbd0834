"""pbsgpu_blob_encode_batch_enc on the GPU (K11 AES-256-GCM + K6 over the ciphertext, with the zstd encoders of every
blob mode): byte for byte equal to tests/crypt_ref.py for host and device bases, decrypted by `cryptography` and decoded
by libzstd (pyarrow's codec), a flipped ciphertext bit fails the tag, inc32 wraps inside a chunk, and a multi-GiB
device batch."""
import os

import numpy as np
import pytest
from cryptography.exceptions import InvalidTag

import crypt_ref
import pbs_plus_b200 as pg
import zstd_lz_ref as lzref
from pbs_plus_b200._lib import EINVAL
from test_gpu_zstd_lz import pack, rnd, to_dev

pytestmark = pytest.mark.gpu
pa = pytest.importorskip("pyarrow")
B = 128 << 10
KEY = bytes(range(7, 39))


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module", autouse=True)
def release_device_memory(torch):
    """The multi-GiB tests' tensors go back to the device when the module is done, not into torch's cache: later
    modules (the full-size cfg2 batch) need nearly all of the HBM free."""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def crypt(eng):
    c = eng.crypt(KEY)
    yield c
    c.close()


def parts():
    """Lengths around the block and segment edges (a segment is 16 KiB), zero runs, text and random bytes."""
    text = lzref.text_corpus(1 << 20, 9)
    return [np.zeros(0, np.uint8), rnd(1, 1), rnd(15, 2), rnd(16, 3), rnd(17, 4), rnd(4095, 5), rnd(16384, 6),
            rnd(16385, 7), rnd(3 * 16384 - 1, 8), rnd((1 << 20) + 3, 9), np.zeros(2 * B + 5, np.uint8),
            np.concatenate([rnd(1000, 10), np.zeros(3 * B, np.uint8), rnd(77, 11)]), text[:300_001], text[5:B + 9]]


def check(key: bytes, blob: bytes, chunk: bytes, mode: str):
    pl, comp = crypt_ref.blob_decrypt(key, blob)
    if comp:
        assert mode != "raw" and len(pl) < len(chunk)
        assert pa.Codec("zstd").decompress(pl, decompressed_size=len(chunk)).to_pybytes() == chunk
    else:
        assert pl == chunk


@pytest.mark.parametrize("mode", ["raw", "z", "lz", "lze", "lzh"])
def test_blob_encode_batch_enc_equals_the_restatement(eng, crypt, torch, mode):
    ps = parts()
    buf, off, ln = pack(ps, 5)
    iv = os.urandom(16 * len(ps))
    want = [crypt_ref.blob_encode_enc(KEY, iv[16 * i:16 * i + 16], p.tobytes(), mode) for i, p in enumerate(ps)]
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = eng.blob_encode_batch_enc(crypt, mode, base, off, ln, iv)
        for i, (b, w, p) in enumerate(zip(blobs, want, ps)):
            assert b == w, (mode, i, len(p))
            assert int(crc[i]) == int.from_bytes(b[8:12], "little")
            check(KEY, b, p.tobytes(), mode)
    # one flipped ciphertext bit: the CRC is recomputed, the tag fails
    i = 9
    bad = bytearray(want[i])
    bad[44 + 1000] ^= 4
    bad[8:12] = __import__("zlib").crc32(bytes(bad[44:])).to_bytes(4, "little")
    with pytest.raises(InvalidTag):
        crypt_ref.blob_decrypt(KEY, bytes(bad))


def test_inc32_wraps_inside_a_chunk(eng, crypt, torch):
    """IVs whose J0 low word is 0xFFFFFFF0, 0xFFFFFFFF or 0: in the first two the counter's low word wraps to 0 inside
    the first segment without a carry into the upper words."""
    js = [0xA5A5A5A5_5A5A5A5A_12345678_FFFFFFF0, 0x01_FFFFFFFF, 0xFFFFFFFF_FFFFFFFF_FFFFFFFF_FFFFFFFF, 0]
    ivs = b"".join(crypt_ref.iv_for_j0(KEY, j) for j in js)
    ps = [rnd((1 << 20) + 9, 20 + k) for k in range(len(js))]
    buf, off, ln = pack(ps, 3)
    blobs, _ = eng.blob_encode_batch_enc(crypt, "raw", to_dev(torch, buf), off, ln, ivs)
    for k, p in enumerate(ps):
        assert blobs[k] == crypt_ref.blob_encode_enc(KEY, ivs[16 * k:16 * k + 16], p.tobytes()), k


def test_two_keys_give_different_blobs_and_bad_arguments_are_refused(eng, crypt, torch):
    p = rnd(5000, 30)
    iv = bytes(16)
    other = eng.crypt(bytes(32))
    a, _ = eng.blob_encode_batch_enc(crypt, "raw", p, [0], [len(p)], iv)
    b, _ = eng.blob_encode_batch_enc(other, "raw", p, [0], [len(p)], iv)
    assert a[0] != b[0] and b[0] == crypt_ref.blob_encode_enc(bytes(32), iv, p.tobytes())
    other.close()
    L = eng._L
    o, l = np.zeros(1, np.uint64), np.full(1, 10, np.uint64)
    out, blen = np.zeros(64, np.uint8), np.zeros(1, np.uint64)
    for mode in (0, 6):   # NONE and out of range
        assert L.pbsgpu_blob_encode_batch_enc(eng._h, crypt._h, mode, p.ctypes.data, o.ctypes.data, l.ctypes.data, 1,
                                              p.ctypes.data, out.ctypes.data, o.ctypes.data, blen.ctypes.data, None) == EINVAL
    with pytest.raises(ValueError):
        eng.blob_encode_batch_enc(crypt, "raw", p, [0], [10], bytes(15))


def test_multi_gib_device_batch(eng, crypt, torch):
    """3 GiB of 4 MiB chunks resident on the device, two of them at odd offsets, every blob checked against AESGCM."""
    n, ch = 3 << 30, 4 << 20
    d = torch.randint(0, 256, (n + 64,), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()   # the library reads d on its own stream
    off = np.arange(0, n - ch, ch, dtype=np.uint64)
    off[1] += 3
    off[-1] += 61
    ln = np.full(len(off), ch, np.uint64)
    ln[-1] -= 7
    iv = os.urandom(16 * len(off))
    blobs, crc = eng.blob_encode_batch_enc(crypt, "raw", d, off, ln, iv)
    host = d.cpu().numpy()
    del d
    torch.cuda.empty_cache()
    for i in range(len(off)):
        o = int(off[i])
        assert blobs[i] == crypt_ref.blob_encode_enc(KEY, iv[16 * i:16 * i + 16], host[o:o + int(ln[i])].tobytes()), i


# ---- keyed digests (K3 with the id_key suffix) -------------------------------------------------------------------
IDENT = crypt_ref.id_key(KEY)


def keyed(parts, rec):
    """rec's records with the keyed digest of every chunk, from the chunk bytes (the cuts are rec's)."""
    out = rec.copy()
    prev = {}
    for r in out:
        s, e = int(r["stream"]), int(r["end_off"])
        b = prev.get(s, 0)
        r["digest"] = np.frombuffer(crypt_ref.compute_digest(parts[s][b:e].tobytes(), IDENT), np.uint8)
        prev[s] = e
    return out


def keyed_parts():
    """Empty, tiny, unaligned starts and streams across several chunks of the 64 KiB chunker."""
    return [np.zeros(0, np.uint8), rnd(1, 40), rnd(63, 41), rnd(64, 42), rnd(120, 43), rnd(70_000, 44),
            rnd(1_000_003, 45), np.zeros(600_000, np.uint8), rnd(3_000_001, 46), lzref.text_corpus(400_000, 3)]


@pytest.fixture(scope="module")
def nopart():
    os.environ["PBSGPU_PARTITION_SMS"] = "0"
    e = pg.Engine(0)
    del os.environ["PBSGPU_PARTITION_SMS"]
    yield e
    e.close()


@pytest.mark.parametrize("partitioned", [True, False])
def test_keyed_digests_of_the_batch_forms(eng, nopart, torch, partitioned):
    import oracle
    e = eng if partitioned else nopart
    c = e.crypt(KEY)
    ps = keyed_parts()
    cfg = pg.make_config(1 << 16)
    plain = oracle.chunk_digest_streams(oracle.config(1 << 16), ps)
    want = keyed(ps, plain)
    assert not (want["digest"] == plain["digest"]).all(axis=1).any()
    buf, off, ln = pack(ps, 3)
    dev = to_dev(torch, buf)
    for base in (buf, dev):
        got = e.chunk_digest_batch(cfg, base, off, ln, crypt=c)
        assert got.tobytes() == want.tobytes()
        assert e.chunk_digest_batch(cfg, base, off, ln).tobytes() == plain.tobytes()
    for early in (False, True):
        got = e.submit(cfg, dev, off, ln, early_input=early, crypt=c).wait()[0]
        assert got.tobytes() == want.tobytes(), early
    got, xxh = e.chunk_digest_batch_xxh3(cfg, buf, off, ln, crypt=c)
    assert got.tobytes() == want.tobytes() and xxh.tolist() == [oracle.xxh3_64(p) for p in ps]
    # the set sees keyed digests: seeded with the keyed digests of the first half, disjoint from the plain ones
    ks = e.digest_set()
    ks.insert(want["digest"][: len(want) // 2])
    got = e.chunk_digest_batch(cfg, dev, off, ln, ks, crypt=c)
    first = {}
    for i, r in enumerate(want):
        first.setdefault(bytes(r["digest"]), i)
    flags = [int(i < len(want) // 2 or first[bytes(r["digest"])] < i) for i, r in enumerate(want)]
    assert got["flags"].tolist() == flags
    assert not {bytes(d) for d in plain["digest"]} & {bytes(d) for d in want["digest"]}
    # sha256_keyed_batch
    d = e.sha256_keyed_batch(c, dev, off, ln)
    assert [bytes(x) for x in d] == [crypt_ref.compute_digest(p.tobytes(), IDENT) for p in ps]
    c.close()


def test_old_batch_opts_size_gives_plain_digests(eng, crypt, torch):
    import ctypes as C
    ps = keyed_parts()
    buf, off, ln = pack(ps, 0)
    cfg = pg.make_config(1 << 16)
    from pbs_plus_b200._lib import CHUNK_DTYPE, BatchOpts
    out = np.zeros(4096, dtype=CHUNK_DTYPE)
    n = C.c_uint64()
    for size, keyed_want in ((48, False), (56, True)):
        o = BatchOpts()
        o.size, o.crypt = size, crypt._h.value
        rc = eng._L.pbsgpu_chunk_digest_batch_ex(eng._h, C.byref(cfg), buf.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                                 len(off), C.byref(o), out.ctypes.data, len(out), C.byref(n))
        assert rc == 0
        plain = eng.chunk_digest_batch(cfg, buf, off, ln)
        got = out[: n.value]
        assert (got.tobytes() == plain.tobytes()) != keyed_want
    o = BatchOpts()
    o.size = 52
    assert eng._L.pbsgpu_chunk_digest_batch_ex(eng._h, C.byref(cfg), buf.ctypes.data, off.ctypes.data, ln.ctypes.data,
                                               len(off), C.byref(o), out.ctypes.data, len(out), C.byref(n)) == EINVAL


def test_keyed_digests_of_a_resident_cfg2_batch(eng, crypt, torch):
    """64 files of the cfg2 corpus (64 MiB each, seed 2, 4 MiB average chunks) resident on the device: the keyed
    records have the plain records' cuts and SHA-256(chunk || id_key) as digests."""
    import hashlib
    n_files, flen = 64, 64 << 20
    dev = torch.empty(n_files * flen, dtype=torch.uint8, device="cuda")
    eng.corpus_fill(pg.corpus(seed=2, file_len=flen), 0, n_files, dev, flen)
    torch.cuda.synchronize()
    off = np.arange(n_files, dtype=np.uint64) * flen
    ln = np.full(n_files, flen, np.uint64)
    cfg = pg.make_config(4 << 20)
    plain = eng.chunk_digest_batch(cfg, dev, off, ln)
    got = eng.submit(cfg, dev, off, ln, early_input=True, crypt=crypt).wait()[0]
    assert (got["end_off"] == plain["end_off"]).all() and (got["stream"] == plain["stream"]).all()
    host = dev.cpu().numpy()
    del dev
    torch.cuda.empty_cache()
    prev = {}
    for r in got:
        s, e = int(r["stream"]), int(r["end_off"])
        b = prev.get(s, 0)
        prev[s] = e
        assert bytes(r["digest"]) == hashlib.sha256(host[s * flen + b: s * flen + e].tobytes() + IDENT).digest()


# ---- the stream and the writers in encrypt mode ----------------------------------------------------------------
def test_stream_with_crypt_equals_the_batch_call(eng, crypt, torch):
    import hashlib
    os.environ["PBSGPU_STREAM_WINDOW"] = str(1 << 20)
    e = pg.Engine(0)
    del os.environ["PBSGPU_STREAM_WINDOW"]
    try:
        c = e.crypt(KEY)
        data = np.concatenate([rnd(2_500_000, 60), np.zeros(700_000, np.uint8), lzref.text_corpus(900_000, 4)])
        cfg = pg.make_config(1 << 16)
        want = e.chunk_digest_batch(cfg, data, [0], [len(data)], crypt=c)
        seed = bytes(range(32))
        for cuts in ([len(data)], [1, 100_000, 1_048_577, 2_000_000, len(data)]):
            s = e.stream(cfg, e.digest_set())
            s.crypt(c, iv_seed=seed)
            s.blob_mode("lzh")
            pos = 0
            for cut in cuts:
                s.write(data[pos:cut])
                pos = cut
            rec = s.finish()
            blobs = s.poll_blobs()
            s.close()
            assert (rec["end_off"] == want["end_off"]).all() and (rec["digest"] == want["digest"]).all()
            new = [k for k in range(len(rec)) if not rec["flags"][k] & 1]
            assert len(blobs) == len(new)
            for k, (i, b) in enumerate(zip(new, blobs)):
                lo = int(rec["end_off"][i - 1]) if i else 0
                iv = hashlib.sha256(seed + k.to_bytes(8, "little")).digest()[:16]
                chunk = data[lo:int(rec["end_off"][i])].tobytes()
                assert b == crypt_ref.blob_encode_enc(KEY, iv, chunk, "lzh"), k
        s = e.stream(cfg)
        s.write(data[:10])
        with pytest.raises(pg.PbsGpuError):
            s.crypt(c)
        s.close()
        c.close()
    finally:
        e.close()


def test_writers_with_a_crypt_key_give_keyed_indexes_and_encrypted_blobs(eng):
    import io
    from pbs_plus_b200 import transfer
    from test_gpu_round2 import _payload_stream
    files = [rnd(n, 70 + i) for i, n in enumerate((0, 100, 300_000, 1_200_000, 77))]
    cfg = pg.make_config(1 << 16)
    got = []
    w = transfer.PayloadStreamWriter(eng, cfg, eng.digest_set(), upload_blob=lambda d, b: got.append((d, b)),
                                     blob_compression="lze", crypt_key=KEY)
    for i, f in enumerate(files):
        w.WriteEntryReader(transfer.Entry(f"f{i}", len(f)), io.BytesIO(f.tobytes()), len(f))
    idx = w.Finish()
    stream, _ = _payload_stream(files)
    prev, chunks = 0, {}
    for end, dig, known in idx:
        ch = stream[prev:end].tobytes()
        assert dig == crypt_ref.compute_digest(ch, IDENT)
        chunks[dig] = ch
        prev = end
    ends, digs = eng.didx_parse(w.didx())
    assert [bytes(d) for d in digs] == [d for _, d, _ in idx]
    assert len(got) == len({d for _, d, known in idx if not known})
    for d, b in got:
        check(KEY, b, chunks[d], "lze")
    # DedupWriter: keyed index records, encrypted blobs
    got = []
    dw = transfer.DedupWriter(eng, cfg, eng.digest_set(), upload_blob=lambda d, b: got.append((d, b)),
                              blob_compression="lzh", crypt_key=KEY)
    for i, f in enumerate(files):
        dw.WriteEntry(transfer.Entry(f"f{i}", len(f)), f.tobytes())
    recs = dw.Finish()
    prev, chunks = {}, {}
    for r in recs:
        f = files[int(r.path[1:])]
        ch = f[prev.get(r.path, 0):r.end_off].tobytes()
        prev[r.path] = r.end_off
        assert r.digest == crypt_ref.compute_digest(ch, IDENT)
        chunks[r.digest] = ch
    assert len(got) == sum(not r.known for r in recs)
    for d, b in got:
        check(KEY, b, chunks[d], "lzh")
