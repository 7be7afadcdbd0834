"""pbsgpu_blob_encode_batch_lzl on the GPU (K8 + K12 + K9 / K10 with long spans): bit-exact against
tests/zstd_ldm_ref.py (blob_encode_lzl), decoded by libzstd (pyarrow's codec), never larger than the _lzh blob of the
same chunk; for a mixed batch, chunker output, a large device batch across pass edges, the stream's blob mode, both
writers and encrypted blobs."""
import io
import os
import zlib

import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg
import crypt_ref
import zstd_huf_ref as hufref
import zstd_ldm_ref as ldm
import zstd_lz_ref as lzref
from oracle import pyref
from pbs_plus_b200 import transfer
from pbs_plus_b200._lib import EINVAL
from test_gpu_round2 import _payload_stream
from test_gpu_stream_blobs import engine, write_stream
from test_gpu_zstd_lz import check_blob, mixed_parts, pack, rnd, to_dev
from test_zstd_ldm_cpu import census_parts, far_copy, ldm_parts, REQUIRED_LZL
import zstd_forms as zf

pytestmark = pytest.mark.gpu
B = pyref.ZFRAME_BLOCK
pa = pytest.importorskip("pyarrow")
KEY = bytes(range(50, 82))


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module", autouse=True)
def release_device_memory(torch):
    """The large batch's tensors go back to the device when the module is done, not into torch's cache."""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


def test_blob_encode_batch_lzl_equals_the_restatement_for_a_mixed_batch(eng, torch):
    """census_parts() (the form cases, the other zstd tests' inputs and the long-match cases), a few mixed chunks and
    copies exactly at and one byte beyond the largest offset, from host and device memory; the census of the GPU's
    own frames covers the lzl forms."""
    parts = census_parts() + mixed_parts()[:6] + [far_copy(ldm.LDM_MAXDIST), far_copy(ldm.LDM_MAXDIST + 1)]
    want = [ldm.blob_encode_lzl(p.tobytes()) for p in parts]
    buf, off, ln = pack(parts, 5)
    smaller = set()
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = eng.blob_encode_batch_lzl(base, off, ln)
        lzh, _ = eng.blob_encode_batch_lzh(base, off, ln)
        for i, (blob, p) in enumerate(zip(blobs, parts)):
            assert blob == want[i], (i, len(p), len(blob), len(want[i]))
            check_blob(blob, p.tobytes(), int(crc[i]))
            assert len(blob) <= len(lzh[i])
            smaller.add(len(blob) < len(lzh[i]))
    assert smaller == {True, False}
    frames = [b[12:] for b in blobs if b[:8] == pyref.BLOB_MAGIC_COMPRESSED]
    c = zf.census(frames)
    assert not REQUIRED_LZL - set(c), sorted(REQUIRED_LZL - set(c))


def repeated_mix(n: int, seed: int) -> np.ndarray:
    """Text and binary data with near-copies of earlier stretches 100 KiB - 3 MiB back."""
    rng = np.random.default_rng(seed)
    base = np.concatenate([hufref.binary_corpus(n // 2, seed), lzref.text_corpus(n - n // 2, seed + 1)])
    out = base.copy()
    for _ in range(n // (256 << 10)):
        ln = int(rng.integers(2000, 200_000))
        dst = int(rng.integers(3 << 20, n - ln))
        src = dst - int(rng.integers(100 << 10, 3 << 20))
        out[dst:dst + ln] = out[src:src + ln]
    out[rng.integers(0, n, n // 2000)] = rng.integers(0, 256, n // 2000, dtype=np.uint8)
    return out


def test_blob_encode_batch_lzl_on_chunker_output(eng, torch):
    """The chunks of an image with far near-copies and a zero run: byte-exact, each at most its _lzh blob, smaller in
    total."""
    img = np.concatenate([repeated_mix(10 << 20, 60), np.zeros(2 << 20, np.uint8), repeated_mix(4 << 20, 61)])
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(4 << 20), d, [0], [len(img)])
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    blobs, crc = eng.blob_encode_batch_lzl(d, starts, ends - starts)
    lzh, _ = eng.blob_encode_batch_lzh(d, starts, ends - starts)
    for k, (s0, e0) in enumerate(zip(starts, ends)):
        chunk = img[int(s0):int(e0)].tobytes()
        assert blobs[k] == ldm.blob_encode_lzl(chunk), k
        check_blob(blobs[k], chunk, int(crc[k]))
        assert len(blobs[k]) <= len(lzh[k])
    assert sum(map(len, blobs)) < 0.9 * sum(map(len, lzh))


def test_blob_encode_batch_lzl_large_device_batch_across_pass_edges(eng, torch):
    """~1 GiB of two alternating chunk contents (4 MiB + 1000 and 4 MiB - 3000 bytes, 4 near-copies of 1 MiB each):
    more than LZ_PASS_BLOCKS blocks and more than LZ_PASS_BLOCKS span blocks, so chunks straddle the pass edges of
    both lists, and many K12 passes.  Every blob equals the restatement of its content."""
    a = ldm.repeated_image(hufref.binary_corpus(1 << 20, 70), 4, 2000, 71)
    a = np.concatenate([a, lzref.text_corpus(1000, 72)])
    b = ldm.repeated_image(lzref.text_corpus(1 << 20, 73), 4, 500, 74)[:(4 << 20) - 3000]
    want = [ldm.blob_encode_lzl(a.tobytes()), ldm.blob_encode_lzl(b.tobytes())]
    assert all(len(w) < 0.4 * len(p) for w, p in zip(want, (a, b)))
    pair = np.concatenate([a, b])
    reps = (1 << 30) // len(pair) + 1
    d = to_dev(torch, pair).repeat(reps)
    torch.cuda.synchronize()                                # the engine's streams do not wait for torch's
    off = np.zeros(2 * reps, np.uint64)
    ln = np.zeros(2 * reps, np.uint64)
    off[0::2] = np.arange(reps, dtype=np.uint64) * np.uint64(len(pair))
    off[1::2] = off[0::2] + np.uint64(len(a))
    ln[0::2], ln[1::2] = len(a), len(b)
    assert (ln + np.uint64(B - 1)).__floordiv__(np.uint64(B)).sum() > 2 * 4096
    blobs, crc = eng.blob_encode_batch_lzl(d, off, ln)
    for k in range(2 * reps):
        assert blobs[k] == want[k % 2], k
        assert int(crc[k]) == int.from_bytes(want[k % 2][8:12], "little")
    check_blob(blobs[0], a.tobytes(), int(crc[0]))
    check_blob(blobs[1], b.tobytes(), int(crc[1]))
    del d


def test_stream_blob_mode_lzl_equals_the_batch_call():
    """64 KiB windows: the stream's blobs equal the batch call's and the restatement's."""
    e = engine(1 << 16)
    try:
        files = [repeated_mix(4 << 20, 80), np.zeros(200_000, np.uint8), ldm_parts()[1], hufref.binary_corpus(190_000, 32)]
        stream, starts = _payload_stream(files)
        avg = 1 << 20
        ref = oracle.chunk_digest_forced(oracle.config(avg), stream, np.array(starts, np.uint64))
        ends = ref["end_off"].astype(np.uint64)
        off = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
        want, _ = e.blob_encode_batch_lzl(stream, off, ends - off)
        st = e.stream(pg.make_config(avg))
        st.blob_mode("lzl")
        rec, blobs = write_stream(st, files, 50_001, True)
        st.close()
        assert rec["end_off"].tolist() == ref["end_off"].tolist()
        assert blobs == want
        for b, o, l in list(zip(blobs, off, ends - off))[::3]:
            assert b == ldm.blob_encode_lzl(stream[int(o):int(o + l)].tobytes())
    finally:
        e.close()


def test_writers_upload_lzl_datablobs(eng):
    avg = 1 << 20
    files = [("disk.img", repeated_mix(6 << 20, 90)), ("copy.bin", ldm_parts()[5]), ("notes.txt", lzref.text_corpus(700_000, 22))]
    blobs = []
    w = transfer.DedupWriter(eng, pg.make_config(avg), eng.digest_set(), upload_blob=lambda d, b: blobs.append((d, b)),
                             blob_compression="lzl")
    for name, data in files:
        w.WriteEntry(transfer.Entry(name, len(data)), data.tobytes())
    w.Finish()
    ref = oracle.chunk_digest_streams(oracle.config(avg), [d for _, d in files])
    want, seen, start = [], set(), {}
    for r in ref:
        i = int(r["stream"]); s0 = start.get(i, 0); e0 = int(r["end_off"]); start[i] = e0
        dg = bytes(r["digest"])
        if dg not in seen:
            seen.add(dg)
            want.append((dg, ldm.blob_encode_lzl(files[i][1][s0:e0].tobytes())))
    assert blobs == want
    up = []
    pw = transfer.PayloadStreamWriter(eng, pg.make_config(avg), eng.digest_set(), upload_blob=lambda d, b: up.append((d, b)),
                                      blob_compression="lzl")
    for name, data in files:
        pw.WriteEntryReader(transfer.Entry(name, len(data)), io.BytesIO(data.tobytes()), len(data))
    pw.Finish()
    assert up
    for dg, blob in up:
        assert blob[:8] in (pyref.BLOB_MAGIC_COMPRESSED, pyref.BLOB_MAGIC_UNCOMPRESSED)
        pl = blob[12:]
        assert int.from_bytes(blob[8:12], "little") == zlib.crc32(pl)
        if blob[:8] == pyref.BLOB_MAGIC_COMPRESSED:
            size = int.from_bytes(pl[5:13], "little")
            pl = pa.Codec("zstd").decompress(pl, decompressed_size=size).to_pybytes()
        assert __import__("hashlib").sha256(pl).digest() == dg
        assert blob == ldm.blob_encode_lzl(pl)


def test_encrypted_lzl_blobs(eng, torch):
    """blob_encode_batch_enc in lzl mode: the payload is blob_encode_lzl's frame where smaller, encrypted as
    crypt_ref states it, and decrypts and decodes to the chunk."""
    crypt = eng.crypt(KEY)
    try:
        ps = ldm_parts()[:4] + [rnd(5000, 3), np.zeros(2 * B + 5, np.uint8)]
        buf, off, ln = pack(ps, 3)
        iv = os.urandom(16 * len(ps))
        for base in (buf, to_dev(torch, buf)):
            blobs, crc = eng.blob_encode_batch_enc(crypt, "lzl", base, off, ln, iv)
            for i, (blob, p) in enumerate(zip(blobs, ps)):
                chunk = p.tobytes()
                fr = ldm.zstd_frame_lzl(chunk)
                comp = len(chunk) > 0 and len(fr) < len(chunk)
                ct, tag = crypt_ref.gcm_encrypt(KEY, iv[16 * i:16 * i + 16], fr if comp else chunk)
                assert blob[44:] == ct and blob[28:44] == tag, i
                pl, c = crypt_ref.blob_decrypt(KEY, blob)
                assert c == comp and int(crc[i]) == zlib.crc32(ct)
                got = pa.Codec("zstd").decompress(pl, decompressed_size=len(chunk)).to_pybytes() if c else pl
                assert got == chunk
    finally:
        crypt.close()


def test_blob_encode_batch_lzl_error_paths_and_mode_6(eng, torch):
    L, h = eng._L, eng._h
    d = to_dev(torch, rnd(1024, 30))
    off = np.zeros(1, np.uint64)
    ln = np.full(1, 100, np.uint64)
    out = np.zeros(1024, np.uint8)
    oo = np.zeros(1, np.uint64)
    ol = np.zeros(1, np.uint64)
    crc = np.zeros(1, np.uint32)
    p = lambda a: a.ctypes.data
    args = [d.data_ptr(), p(off), p(ln), 1, p(out), p(oo), p(ol), p(crc)]
    assert L.pbsgpu_blob_encode_batch_lzl(h, *args) == 0
    assert out[:8].tobytes() == pyref.BLOB_MAGIC_UNCOMPRESSED and int(ol[0]) == 112
    assert L.pbsgpu_blob_encode_batch_lzl(None, *args) == EINVAL
    for k in (0, 1, 2, 4, 5, 6):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_encode_batch_lzl(h, *bad) == EINVAL, k
    big = np.full(1, 1 << 40, np.uint64)
    assert L.pbsgpu_blob_encode_batch_lzl(h, d.data_ptr(), p(off), p(big), 1, p(out), p(oo), p(ol), p(crc)) == EINVAL
    assert L.pbsgpu_blob_encode_batch_lzl(h, None, None, None, 0, None, None, None, None) == 0
    blobs, crc2 = eng.blob_encode_batch_lzl(d, [], [])
    assert blobs == [] and len(crc2) == 0
    # mode 6 is not assigned: every call that takes a mode refuses it, and 7 is lzl
    crypt = eng.crypt(KEY)
    try:
        hp = rnd(100, 31)
        blen = np.zeros(1, np.uint64)
        for mode, rc in ((6, EINVAL), (8, EINVAL), (7, 0)):
            assert L.pbsgpu_blob_encode_batch_enc(h, crypt._h, mode, hp.ctypes.data, p(off), p(ln), 1, hp.ctypes.data,
                                                  p(out), p(oo), p(blen), None) == rc, mode
    finally:
        crypt.close()
    st = eng.stream(pg.make_config(1 << 16))
    try:
        assert L.pbsgpu_stream_blob_mode(st._h, 6) == EINVAL
        assert L.pbsgpu_stream_blob_mode(st._h, 8) == EINVAL
        assert L.pbsgpu_stream_blob_mode(st._h, 7) == 0
        with pytest.raises(ValueError):
            st.blob_mode("lzx")
    finally:
        st.close()
    with pytest.raises(ValueError):
        eng.blob_encode_batch_enc(eng, "lzx", hp, [0], [10], bytes(16))
    with pytest.raises(ValueError):
        transfer.DedupWriter(eng, pg.make_config(1 << 16), blob_compression="lzx")
