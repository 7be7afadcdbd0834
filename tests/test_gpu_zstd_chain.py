"""pbsgpu_blob_encode_batch_lzc on the GPU (K8 + K16 + K9b / K10): bit-exact against tests/zstd_chain_ref.py
(blob_encode_lzc) for host and device bases, through the encrypted batch call, the payload stream with and without
fixed IVs, the writer, and a call of several K16 passes; every blob goes back through the GPU decoder with its digest;
the census of the GPU's own frames covers REQUIRED_LZC."""
import hashlib
import os
import zlib

import numpy as np
import pytest

import crypt_ref
import oracle
import pbs_plus_b200 as pg
import zstd_chain_ref as ch
import zstd_forms as zf
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from oracle import pyref
from pbs_plus_b200 import transfer
from pbs_plus_b200._lib import DEC_OK, EINVAL
from test_gpu_round2 import _payload_stream
from test_gpu_stream_blobs import engine, write_stream
from test_gpu_zstd_lz import check_blob, pack, rnd, to_dev
from test_zstd_chain_cpu import REQUIRED_LZC, census_parts
from test_zstd_ldm_cpu import far_copy

pytestmark = pytest.mark.gpu
KEY = bytes(range(90, 122))
LZC = 10                      # PBSGPU_BLOB_LZC
PASS_BYTES = 128 << 20        # CH_PASS_BYTES in csrc/zchain.cuh


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module", autouse=True)
def release_device_memory(torch):
    """The multi-pass batch's tensors go back to the device when the module is done, not into torch's cache."""
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
def parts():
    return census_parts() + [far_copy(ch.CH_MAXDIST), far_copy(ch.CH_MAXDIST + 1), lzref.text_corpus(1 << 20, 1),
                             hufref.binary_corpus(600_000, 2)]


@pytest.fixture(scope="module")
def want(parts):
    return [ch.blob_encode_lzc(p.tobytes()) for p in parts]


def decode_back(eng, blobs, chunks, crypt=None):
    """Every blob through pbsgpu_blob_decode_batch (or _enc with crypt) with its digest: status OK, bytes equal."""
    if crypt is None:
        dig = b"".join(hashlib.sha256(c).digest() for c in chunks)
        st, data, _ = eng.blob_decode_batch(blobs, [len(c) for c in chunks], dig)
    else:
        ik = crypt_ref.id_key(KEY)
        dig = b"".join(crypt_ref.compute_digest(c, ik) for c in chunks)
        st, data, _ = eng.blob_decode_batch_enc(crypt, blobs, [len(c) for c in chunks], dig)
    assert (st == DEC_OK).all(), st.tolist()
    assert [bytes(d) for d in data] == list(chunks)


def test_blob_encode_batch_lzc_equals_the_restatement(eng, torch, parts, want):
    """The CPU test's parts, the tests/zstd_forms.py parts, copies exactly at and one byte beyond CH_MAXDIST in 16 MiB
    chunks and the corpora, from host and device memory; the census of the GPU's frames covers REQUIRED_LZC."""
    buf, off, ln = pack(parts, 9)
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = eng.blob_encode_batch_lzc(base, off, ln)
        for i, (blob, p) in enumerate(zip(blobs, parts)):
            assert blob == want[i], (i, len(p), len(blob), len(want[i]))
            check_blob(blob, p.tobytes(), int(crc[i]))
        decode_back(eng, blobs, [p.tobytes() for p in parts])
    c = zf.census([b[12:] for b in blobs if b[:8] == pyref.BLOB_MAGIC_COMPRESSED])
    assert not REQUIRED_LZC - set(c), sorted(REQUIRED_LZC - set(c))


def test_encrypted_lzc_blobs(eng, torch, parts, want):
    """pbsgpu_blob_encode_batch_enc(PBSGPU_BLOB_LZC) with fixed IVs: the payload is blob_encode_lzc's frame where
    smaller, AES-256-GCM as crypt_ref states it; each blob decrypts and decodes on the GPU to its chunk."""
    crypt = eng.crypt(KEY)
    try:
        iv = bytes(np.random.default_rng(5).integers(0, 256, 16 * len(parts), dtype=np.uint8))
        buf, off, ln = pack(parts, 3)
        for base in (buf, to_dev(torch, buf)):
            blobs, crc = eng.blob_encode_batch_enc(crypt, "lzc", base, off, ln, iv)
            for i, (blob, p) in enumerate(zip(blobs, parts)):
                chunk = p.tobytes()
                comp = want[i][:8] == pyref.BLOB_MAGIC_COMPRESSED
                ct, tag = crypt_ref.gcm_encrypt(KEY, iv[16 * i:16 * i + 16], want[i][12:])
                assert blob[12:28] == iv[16 * i:16 * i + 16] and blob[28:44] == tag and blob[44:] == ct, i
                pl, c = crypt_ref.blob_decrypt(KEY, blob)
                assert c == comp and int(crc[i]) == zlib.crc32(ct) == int.from_bytes(blob[8:12], "little")
            decode_back(eng, blobs, [p.tobytes() for p in parts], crypt)
    finally:
        crypt.close()


def test_stream_blob_mode_lzc(eng):
    """64 KiB windows: the stream's blobs equal the batch call's and the restatement's; with a crypt and a fixed
    iv_seed they equal the encrypted restatement."""
    e = engine(1 << 16)
    try:
        files = [lzref.text_corpus(900_000, 80), np.zeros(200_000, np.uint8), hufref.binary_corpus(300_000, 81),
                 ch.half_zero(250_000, 82)]
        stream, starts = _payload_stream(files)
        avg = 1 << 18
        ref = oracle.chunk_digest_forced(oracle.config(avg), stream, np.array(starts, np.uint64))
        ends = ref["end_off"].astype(np.uint64)
        off = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
        chunks = [stream[int(o):int(o + l)].tobytes() for o, l in zip(off, ends - off)]
        st = e.stream(pg.make_config(avg))
        st.blob_mode("lzc")
        rec, blobs = write_stream(st, files, 50_001, True)
        st.close()
        assert rec["end_off"].tolist() == ref["end_off"].tolist()
        assert blobs == [ch.blob_encode_lzc(c) for c in chunks]
        batch, _ = e.blob_encode_batch_lzc(stream, off, ends - off)
        assert blobs == batch
        decode_back(e, blobs, chunks)
        crypt = e.crypt(KEY)
        try:
            seed = bytes(range(32))
            st = e.stream(pg.make_config(avg))
            st.crypt(crypt, iv_seed=seed)
            st.blob_mode("lzc")
            rec, blobs = write_stream(st, files, 70_003, False)
            st.close()
            assert rec["end_off"].tolist() == ref["end_off"].tolist()
            assert len(blobs) == len(chunks)
            for k, (b, c) in enumerate(zip(blobs, chunks)):
                iv = hashlib.sha256(seed + k.to_bytes(8, "little")).digest()[:16]
                ct, tag = crypt_ref.gcm_encrypt(KEY, iv, ch.blob_encode_lzc(c)[12:])
                assert b[12:28] == iv and b[28:44] == tag and b[44:] == ct, k
            decode_back(e, blobs, chunks, crypt)
        finally:
            crypt.close()
    finally:
        e.close()


def test_dedup_writer_uploads_lzc_datablobs(eng):
    avg = 1 << 18
    files = [("notes.txt", lzref.text_corpus(700_000, 22)), ("tool.bin", hufref.binary_corpus(500_000, 23))]
    blobs = []
    w = transfer.DedupWriter(eng, pg.make_config(avg), eng.digest_set(), upload_blob=lambda d, b: blobs.append((d, b)),
                             blob_compression="lzc")
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
            want.append((dg, ch.blob_encode_lzc(files[i][1][s0:e0].tobytes())))
    assert blobs == want


def test_a_call_of_several_passes(eng, torch):
    """~300 MiB of two alternating chunk contents (1 MiB + 1000 bytes of text, 1 MiB - 3000 bytes of binary data):
    three K16 passes of CH_PASS_BYTES, whose first blocks are not at pass position 0 of the call.  Every blob equals
    the restatement of its content and decodes on the GPU."""
    a = lzref.text_corpus((1 << 20) + 1000, 30)
    b = hufref.binary_corpus((1 << 20) - 3000, 31)
    want = [ch.blob_encode_lzc(a.tobytes()), ch.blob_encode_lzc(b.tobytes())]
    pair = np.concatenate([a, b])
    reps = (300 << 20) // len(pair)
    d = to_dev(torch, pair).repeat(reps)
    torch.cuda.synchronize()                                # the engine's streams do not wait for torch's
    off = np.zeros(2 * reps, np.uint64)
    ln = np.zeros(2 * reps, np.uint64)
    off[0::2] = np.arange(reps, dtype=np.uint64) * np.uint64(len(pair))
    off[1::2] = off[0::2] + np.uint64(len(a))
    ln[0::2], ln[1::2] = len(a), len(b)
    assert int(ln.sum()) > 2 * PASS_BYTES
    blobs, crc = eng.blob_encode_batch_lzc(d, off, ln)
    for k in range(2 * reps):
        assert blobs[k] == want[k % 2], k
        assert int(crc[k]) == int.from_bytes(want[k % 2][8:12], "little")
    decode_back(eng, blobs[:4] + blobs[-4:], [a.tobytes(), b.tobytes()] * 4)
    del d


def test_blob_encode_batch_lzc_error_paths(eng, torch):
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
    assert L.pbsgpu_blob_encode_batch_lzc(h, *args) == 0
    assert out[:8].tobytes() == pyref.BLOB_MAGIC_UNCOMPRESSED and int(ol[0]) == 112
    assert L.pbsgpu_blob_encode_batch_lzc(None, *args) == EINVAL
    for k in (0, 1, 2, 4, 5, 6):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_encode_batch_lzc(h, *bad) == EINVAL, k
    big = np.full(1, 1 << 32, np.uint64)   # K16 numbers positions in 32 bits
    assert L.pbsgpu_blob_encode_batch_lzc(h, d.data_ptr(), p(off), p(big), 1, p(out), p(oo), p(ol), p(crc)) == EINVAL
    assert L.pbsgpu_blob_encode_batch_lzc(h, None, None, None, 0, None, None, None, None) == 0
    crypt = eng.crypt(KEY)
    try:
        hp = rnd(100, 31)
        blen = np.zeros(1, np.uint64)
        assert L.pbsgpu_blob_encode_batch_enc(h, crypt._h, LZC, hp.ctypes.data, p(off), p(ln), 1, hp.ctypes.data,
                                              p(out), p(oo), p(blen), None) == 0
    finally:
        crypt.close()
    st = eng.stream(pg.make_config(1 << 16))
    try:
        assert L.pbsgpu_stream_blob_mode(st._h, LZC) == 0
    finally:
        st.close()
