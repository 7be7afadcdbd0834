"""pbsgpu_blob_decode_batch_enc on the GPU (K6 + K11 decrypt + K13 + keyed K3): encrypted blobs of every mode, libzstd
frames and raw chunks encrypted by the restatement, and GCM's edges decode to their chunks with keyed digests, from
host and device bases into host, device or no output; every status, with no byte of a rejected blob reaching `out`;
seeded corruption never passes; plain and encrypted blobs mix; the writers' uploads verify against their indexes; and a
~2.3 GiB batch crosses the pass edges."""
import random
import zlib

import numpy as np
import pytest

import crypt_ref
import zstd_dec_forms as zd
import zstd_forms as zf
import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib
from pbs_plus_b200.engine import _ptr
from test_gpu_blob_decode import sha, zblob
from test_gpu_zstd_lz import pack, rnd, to_dev
from test_zstd_decode_cpu import corpora, libzstd_payloads

pytestmark = pytest.mark.gpu
pa = pytest.importorskip("pyarrow")
KEY = bytes(range(101, 133))
IDENT = crypt_ref.id_key(KEY)
ENCRYPTED = crypt_ref.ENCRYPTED_BLOB_MAGIC_1_0
ENCR_COMPR = crypt_ref.ENCR_COMPR_BLOB_MAGIC_1_0
REJECTED = (_lib.DEC_BAD_MAGIC, _lib.DEC_BAD_CRC, _lib.DEC_BAD_TAG)


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


@pytest.fixture(scope="module")
def crypt(eng):
    c = eng.crypt(KEY)
    yield c
    c.close()


def keyed(c: bytes) -> bytes:
    return crypt_ref.compute_digest(c, IDENT)


def enc_blob(payload: bytes, iv: bytes, magic: bytes) -> bytes:
    """An encrypted blob of any payload (libzstd frames, a raw chunk), built by the restatement."""
    ct, tag = crypt_ref.gcm_encrypt(KEY, iv, payload)
    return magic + zlib.crc32(ct).to_bytes(4, "little") + iv + tag + ct


def ivs(n: int, seed: int) -> bytes:
    return random.Random(seed).randbytes(16 * n)


def check(eng, crypt, blobs, chunks, torch, digests=None):
    """Host blobs into host / device / no output, and the same blobs at ragged offsets of a device buffer into device
    / no output: all OK, bytes equal, digests equal to `digests` (keyed by default)."""
    want = np.frombuffer(b"".join(digests or [keyed(c) for c in chunks]), np.uint8).reshape(-1, 32)
    lens = [len(c) for c in chunks]
    bb, bo, bl = pack([np.frombuffer(b, np.uint8) for b in blobs], 7)
    dev = (to_dev(torch, bb), bo, bl)
    for src, outs in ((blobs, ("host", "device", None)), (dev, ("device", None))):
        for out in outs:
            st, data, dig = eng.blob_decode_batch_enc(crypt, src, lens, digests=want.tobytes(), out=out)
            assert (st == _lib.DEC_OK).all(), (out, st.tolist())
            assert (dig == want).all(), out
            if out is not None:
                for k, c in enumerate(chunks):
                    got = data[k] if out == "host" else data[k].cpu().numpy().tobytes()
                    assert got == c, (out, k)


@pytest.mark.parametrize("mode", ["raw", "z", "lz", "lze", "lzh", "lzl"])
def test_round_trip_of_every_mode_on_the_form_cases(eng, crypt, torch, mode):
    parts = [p for p, _ in zf.form_cases()] + [np.zeros(3 << 17, np.uint8)]   # zero blocks: every mode compresses one
    buf, off, ln = pack(parts, 5)
    blobs, _ = eng.blob_encode_batch_enc(crypt, mode, buf, off, ln, ivs(len(parts), 1))
    if mode != "raw":
        assert any(b[:8] == ENCR_COMPR for b in blobs)
    check(eng, crypt, blobs, [p.tobytes() for p in parts], torch)


def test_round_trip_of_every_mode_on_chunker_output_verify_only(eng, crypt, torch):
    img = np.concatenate([corpora(6 << 20, 3)["text"], np.zeros(1 << 20, np.uint8), corpora(5 << 20, 4)["binary"]])
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), d, [0], [len(img)], crypt=crypt)
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    assert bytes(rec["digest"][0]) == keyed(img[:int(ends[0])].tobytes())
    for mode in ("raw", "z", "lz", "lze", "lzh", "lzl"):
        blobs, _ = eng.blob_encode_batch_enc(crypt, mode, d, starts, ends - starts, ivs(len(ends), 2))
        st, data, dig = eng.blob_decode_batch_enc(crypt, blobs, ends - starts, digests=rec["digest"].tobytes(), out=None)
        assert data is None and (st == _lib.DEC_OK).all(), mode
        assert (dig == rec["digest"]).all(), mode


def test_foreign_encryptions_of_libzstd_frames_fixture_frames_and_a_raw_chunk(eng, crypt, torch):
    items = libzstd_payloads(1 << 20, 5)
    payloads = [p for _, _, p, _ in items]
    chunks = [c for _, _, _, c in items]
    for p, c in zd.fixture_cases().values():
        payloads.append(p)
        chunks.append(c)
    iv = ivs(len(payloads) + 1, 3)
    blobs = [enc_blob(p, iv[16 * k:16 * k + 16], ENCR_COMPR) for k, p in enumerate(payloads)]
    raw = corpora(300_001, 6)["binary"].tobytes()
    blobs.append(enc_blob(raw, iv[-16:], ENCRYPTED))
    chunks.append(raw)
    check(eng, crypt, blobs, chunks, torch)


def test_gcm_edges_and_an_inc32_wrap(eng, crypt, torch):
    """Payloads around the block and the 16 KiB segment edges, and IVs whose counter's low word wraps inside the payload."""
    sizes = [0, 1, 15, 16, 17, 16383, 16384, 16385, 3 * 16384 + 7]
    chunks = [rnd(s, 40 + s % 97).tobytes() for s in sizes]
    iv = ivs(len(sizes), 4)
    blobs = [crypt_ref.blob_encode_enc(KEY, iv[16 * k:16 * k + 16], c) for k, c in enumerate(chunks)]
    for j0 in (0xA5A5A5A5_5A5A5A5A_12345678_FFFFFFF0, 0x01_FFFFFFFF, (1 << 128) - 1):
        c = rnd((1 << 20) + 9, j0 & 0xFFFF).tobytes()
        blobs.append(crypt_ref.blob_encode_enc(KEY, crypt_ref.iv_for_j0(KEY, j0), c))
        chunks.append(c)
    # ENCR_COMPR blobs of the same lengths' libzstd frames
    text = corpora(100_000, 8)["text"].tobytes()
    for s in (17, 16385):
        fr = pa.Codec("zstd", compression_level=1).compress(text[:s], asbytes=True)
        blobs.append(enc_blob(fr, bytes([s & 255]) * 16, ENCR_COMPR))
        chunks.append(text[:s])
    check(eng, crypt, blobs, chunks, torch)


def corrupt_checksum_frame():
    """checksum_raw's frame with a byte inside its first Raw_Block flipped: only the content checksum sees it."""
    ck_payload, ck_data = zd.fixture_cases()["checksum_raw"]
    fr = zd.split_payload(ck_payload)[0][1]
    fhd = fr[4]
    p = 5 + (not (fhd >> 5) & 1) + ((1 if (fhd >> 5) & 1 else 0), 2, 4, 8)[fhd >> 6]
    while True:
        h = int.from_bytes(fr[p:p + 3], "little")
        if (h >> 1) & 3 == 0:
            break
        p += 3 + (1 if (h >> 1) & 3 == 1 else h >> 3)
    flipped = bytearray(ck_payload)
    flipped[p + 3 + 100] ^= 0x40
    return bytes(flipped), ck_data


def recrc(b: bytearray) -> bytes:
    b[8:12] = zlib.crc32(bytes(b[44:])).to_bytes(4, "little")
    return bytes(b)


def call_raw(eng, crypt_h, blobs, lens, digests, out, out_off):
    """pbsgpu_blob_decode_batch_enc with the caller's own `out` (a pre-filled host array or device tensor)."""
    L = eng._L
    base = np.frombuffer(b"".join(blobs), np.uint8)
    o = np.zeros(len(blobs), np.uint64)
    o[1:] = np.cumsum([len(b) for b in blobs])[:-1]
    l = np.array([len(b) for b in blobs], np.uint64)
    cl = np.array(lens, np.uint64)
    st = np.zeros(len(blobs), np.int32)
    rc = L.pbsgpu_blob_decode_batch_enc(eng._h, crypt_h, base.ctypes.data, o.ctypes.data, l.ctypes.data, len(blobs),
                                        cl.ctypes.data, digests.ctypes.data, _ptr(out), out_off.ctypes.data,
                                        st.ctypes.data, None)
    assert rc == 0
    return st


def test_per_blob_statuses_and_no_rejected_byte_reaches_out(eng, crypt, torch):
    text = corpora(300_000, 9)["text"].tobytes()
    iv = ivs(16, 5)
    good = crypt_ref.blob_encode_enc(KEY, iv[:16], text)
    frame = pa.Codec("zstd", compression_level=3).compress(text, asbytes=True)
    good_c = enc_blob(frame, iv[16:32], ENCR_COMPR)
    ck_frame, ck_data = corrupt_checksum_frame()
    tag_flip, iv_flip, ct_flip, crc_flip = bytearray(good), bytearray(good), bytearray(good), bytearray(good)
    tag_flip[30] ^= 0x10
    iv_flip[13] ^= 0x01
    ct_flip[44 + 5000] ^= 0x80
    crc_flip[44 + 7] ^= 0x02
    cases = [  # (blob, chunk, chunk_len, digest given, status)
        (good, text, len(text), keyed(text), _lib.DEC_OK),
        (b"\0" * 8 + good[8:], text, len(text), keyed(text), _lib.DEC_BAD_MAGIC),
        (ENCRYPTED + good[8:40], text, len(text), keyed(text), _lib.DEC_BAD_MAGIC),
        (bytes(crc_flip), text, len(text), keyed(text), _lib.DEC_BAD_CRC),
        (bytes(tag_flip), text, len(text), keyed(text), _lib.DEC_BAD_TAG),
        (recrc(iv_flip), text, len(text), keyed(text), _lib.DEC_BAD_TAG),
        (recrc(ct_flip), text, len(text), keyed(text), _lib.DEC_BAD_TAG),
        (enc_blob(b"\x28\xb5\x2f\xfd\x00", iv[32:48], ENCR_COMPR), b"", 0, keyed(b""), _lib.DEC_BAD_FRAME),
        (good, text, len(text) + 1, keyed(text), _lib.DEC_BAD_SIZE),
        (enc_blob(ck_frame, iv[48:64], ENCR_COMPR), ck_data, len(ck_data), keyed(ck_data), _lib.DEC_BAD_CHECKSUM),
        (good_c, text, len(text), sha(text), _lib.DEC_BAD_DIGEST),
        (good_c, text, len(text), keyed(text), _lib.DEC_OK),
        (zblob(frame), text, len(text), sha(text), _lib.DEC_OK),   # plain blobs keep plain digests
    ]
    blobs, chunks, lens, digs, want = (list(x) for x in zip(*cases))
    # between intact neighbours
    nb = good_c
    blobs = [x for b in blobs for x in (nb, b)] + [nb]
    lens = [x for l in lens for x in (len(text), l)] + [len(text)]
    digs = [x for d in digs for x in (keyed(text), d)] + [keyed(text)]
    want = [x for w in want for x in (_lib.DEC_OK, w)] + [_lib.DEC_OK]
    dg = np.frombuffer(b"".join(digs), np.uint8)
    for out in ("host", "device", None):
        st, data, _ = eng.blob_decode_batch_enc(crypt, blobs, lens, digests=dg.tobytes(), out=out)
        assert st.tolist() == want, out
    # the plain call still says ENCRYPTED
    st, _, _ = eng.blob_decode_batch(blobs, lens, out=None)
    assert all(s == _lib.DEC_ENCRYPTED for s, b in zip(st, blobs) if b[:8] in (ENCRYPTED, ENCR_COMPR) and len(b) >= 12)
    # a second key: every encrypted blob fails its tag, the plain one still decodes
    other = eng.crypt(bytes(32))
    st, _, _ = eng.blob_decode_batch_enc(other, blobs, lens, out=None)
    other.close()
    assert st.tolist() == [w if w in (_lib.DEC_BAD_MAGIC, _lib.DEC_BAD_CRC) else
                           _lib.DEC_BAD_TAG if b[:8] in (ENCRYPTED, ENCR_COMPR) else _lib.DEC_OK for b, w in zip(blobs, want)]
    # the caller's `out`, pre-filled: the regions of rejected blobs keep the sentinel
    ooff = np.zeros(len(blobs), np.uint64)
    ooff[1:] = np.cumsum(lens)[:-1]
    total = int(sum(lens))
    host = np.full(total, 0xA5, np.uint8)
    dev = torch.full((total,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for out in (host, dev):
        st = call_raw(eng, crypt._h, blobs, lens, dg, out, ooff)
        assert st.tolist() == want
        got = out if isinstance(out, np.ndarray) else out.cpu().numpy()
        for k, s in enumerate(st):
            region = got[int(ooff[k]): int(ooff[k]) + lens[k]]
            if s in REJECTED:
                assert (region == 0xA5).all(), (k, s)
            elif s in (_lib.DEC_OK, _lib.DEC_BAD_DIGEST):
                assert region.tobytes() == (text if k % 2 == 0 else chunks[k // 2]), k


def test_seeded_corruption_never_decodes(eng, crypt, torch):
    """300 bit flips over the IV, the tag and the ciphertext, the CRC recomputed, each between intact neighbours."""
    rng = random.Random(77)
    text = corpora(200_000, 11)["text"].tobytes()
    frame = pa.Codec("zstd", compression_level=5).compress(text, asbytes=True)
    srcs = [crypt_ref.blob_encode_enc(KEY, rng.randbytes(16), text[:70_001]), enc_blob(frame, rng.randbytes(16), ENCR_COMPR)]
    lens_of = [70_001, len(text)]
    blobs, lens, which = [srcs[1]], [len(text)], []
    for k in range(300):
        s = k % 2
        b = bytearray(srcs[s])
        region = rng.choice(((12, 28), (28, 44), (44, len(b))))
        pos = rng.randrange(*region)
        b[pos] ^= 1 << rng.randrange(8)
        blobs += [recrc(b), srcs[1]]
        lens += [lens_of[s], len(text)]
        which.append(pos)
    st, _, _ = eng.blob_decode_batch_enc(crypt, blobs, lens, out=None)
    assert (st[0::2] == _lib.DEC_OK).all()
    assert (st[1::2] == _lib.DEC_BAD_TAG).all(), [(p, s) for p, s in zip(which, st[1::2]) if s != _lib.DEC_BAD_TAG][:5]


def test_mixed_batch_plain_and_encrypted(eng, crypt, torch):
    parts = [corpora(400_000, 12)["text"], rnd(70_000, 13), np.zeros(300_000, np.uint8), corpora(500_000, 14)["binary"]]
    buf, off, ln = pack(parts, 3)
    plain, _ = eng.blob_encode_batch_lzh(buf, off, ln)
    enc, _ = eng.blob_encode_batch_enc(crypt, "lzh", buf, off, ln, ivs(len(parts), 6))
    blobs, chunks, digs = [], [], []
    for k, p in enumerate(parts):
        c = p.tobytes()
        blobs += [plain[k], enc[k]]
        chunks += [c, c]
        digs += [sha(c), keyed(c)]
    check(eng, crypt, blobs, chunks, torch, digests=digs)
    st, _, _ = eng.blob_decode_batch(blobs, [len(c) for c in chunks], out=None)
    assert st.tolist() == [_lib.DEC_OK, _lib.DEC_ENCRYPTED] * len(parts)


def test_stream_writer_uploads_verify_against_its_index(eng, crypt):
    import io
    from pbs_plus_b200 import transfer
    from test_gpu_round2 import _payload_stream
    files = [rnd(n, 80 + i) for i, n in enumerate((0, 100, 300_000, 1_200_000, 77))]
    files.append(np.tile(corpora(200_000, 15)["text"], 3))
    got = {}
    w = transfer.PayloadStreamWriter(eng, pg.make_config(1 << 16), eng.digest_set(),
                                     upload_blob=lambda d, b: got.setdefault(bytes(d), b), blob_compression="lzh",
                                     crypt_key=KEY)
    for i, f in enumerate(files):
        w.WriteEntryReader(transfer.Entry(f"f{i}", len(f)), io.BytesIO(f.tobytes()), len(f))
    idx = w.Finish()
    prev, blobs, lens, digs = 0, [], [], []
    for end, dig, _ in idx:
        blobs.append(got[bytes(dig)])
        lens.append(end - prev)
        digs.append(bytes(dig))
        prev = end
    st, data, dout = eng.blob_decode_batch_enc(crypt, blobs, lens, digests=b"".join(digs), out="host")
    assert (st == _lib.DEC_OK).all()
    stream, _ = _payload_stream(files)
    assert b"".join(data) == stream.tobytes()
    # the same through the dynamic index image
    ends, idg = eng.didx_parse(w.didx())
    clen = np.diff(np.concatenate([[0], ends])).astype(np.uint64)
    st, _, dout = eng.blob_decode_batch_enc(crypt, [got[bytes(d)] for d in idg], clen, digests=idg.tobytes(), out=None)
    assert (st == _lib.DEC_OK).all() and (dout == idg).all()


def test_a_2_gib_encrypted_batch_crosses_the_pass_edges(eng, crypt, torch):
    """590 encrypted blobs of 4 MiB (2.3 GiB of ciphertext, more than one pass of ZDEC_PASS_BYTES), verify only, from a
    host base."""
    n, size = 590, 4 << 20
    d = torch.empty(n * size, dtype=torch.uint8, device="cuda")
    eng.corpus_fill(pg.corpus(seed=23, file_len=size, run_blocks=4), 0, n, d, size)
    d.view(n, size)[::3, : 1 << 20] = 0                  # zero runs: every third blob is ENCR_COMPR
    torch.cuda.synchronize()
    off = np.arange(n, dtype=np.uint64) * size
    ln = np.full(n, size, np.uint64)
    want = eng.sha256_keyed_batch(crypt, d, off, ln)
    buf = np.zeros(n * (size + 44), np.uint8)
    boff, blen, pos = np.zeros(n, np.uint64), np.zeros(n, np.uint64), 0
    q = (n + 3) // 4
    for g in range(0, n, q):
        blobs, _ = eng.blob_encode_batch_enc(crypt, "z", d, off[g:g + q], ln[g:g + q], ivs(len(off[g:g + q]), g))
        for k, b in enumerate(blobs):
            buf[pos:pos + len(b)] = np.frombuffer(b, np.uint8)
            boff[g + k], blen[g + k] = pos, len(b)
            pos += len(b)
        del blobs
    del d
    torch.cuda.empty_cache()
    assert int((blen - 44).sum()) > 2 << 30 and (blen < size + 44).sum() >= n // 3
    st, data, dig = eng.blob_decode_batch_enc(crypt, (buf, boff, blen), ln, digests=want.tobytes(), out=None)
    assert data is None and (st == _lib.DEC_OK).all() and (dig == want).all()


def test_bad_arguments(eng, crypt):
    L, h = eng._L, eng._h
    text = b"x" * 1000
    good = np.frombuffer(crypt_ref.blob_encode_enc(KEY, bytes(16), text), np.uint8)
    o, l, cl = (np.array([x], np.uint64) for x in (0, len(good), len(text)))
    st = np.zeros(1, np.int32)
    args = [h, crypt._h, good.ctypes.data, o.ctypes.data, l.ctypes.data, 1, cl.ctypes.data, None, None, None, st.ctypes.data,
            None]
    assert L.pbsgpu_blob_decode_batch_enc(*args) == 0 and st[0] == _lib.DEC_OK
    for k in (0, 1, 2, 3, 4, 6, 10):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_decode_batch_enc(*bad) == _lib.EINVAL, k
    outb = np.zeros(len(text), np.uint8)
    bad = list(args)
    bad[8] = outb.ctypes.data          # out without out_off
    assert L.pbsgpu_blob_decode_batch_enc(*bad) == _lib.EINVAL
    big = np.array([1 << 32], np.uint64)
    bad = list(args)
    bad[6] = big.ctypes.data
    assert L.pbsgpu_blob_decode_batch_enc(*bad) == _lib.EINVAL
    e2 = pg.Engine(0)                  # a crypt handle of another context
    c2 = e2.crypt(KEY)
    bad = list(args)
    bad[1] = c2._h
    assert L.pbsgpu_blob_decode_batch_enc(*bad) == _lib.EINVAL
    c2.close()
    e2.close()
    with pytest.raises(pg.PbsGpuError):
        eng.blob_decode_batch_enc(None, [bytes(good)], [len(text)])
    assert L.pbsgpu_blob_decode_batch_enc(h, crypt._h, None, None, None, 0, None, None, None, None, None, None) == 0
