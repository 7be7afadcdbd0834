"""pbsgpu_blob_decode_batch on the GPU (K6 + K13 + K3): every encoder's blobs and libzstd's frames decode to their
chunks with the right digests, from host and device bases into host, device or no output; an index drives a verify
end to end; every per-blob status; corrupted frames never pass where libzstd fails and never decode to other bytes;
and a ~4 GiB batch crosses the decoder's pass edges."""
import hashlib
import random
import zlib

import numpy as np
import pytest

from oracle import pyref
import zstd_dec_forms as zd
import zstd_forms as zf
import zstd_stream_ref
import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib
from test_gpu_zstd_lz import pack, to_dev
from test_zstd_decode_cpu import corpora, libzstd_payloads

pytestmark = pytest.mark.gpu
pa = pytest.importorskip("pyarrow")
ENCRYPTED = bytes([0x7B, 0x67, 0x85, 0xBE, 0x22, 0x2D, 0x4C, 0xF0])
ENCR_COMPR = bytes([0xE6, 0x59, 0x1B, 0xBF, 0x0B, 0xBF, 0xD8, 0x0B])


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


def zblob(payload: bytes) -> bytes:
    return pyref.BLOB_MAGIC_COMPRESSED + zlib.crc32(payload).to_bytes(4, "little") + payload


def sha(b: bytes) -> bytes:
    return hashlib.sha256(b).digest()


def check(eng, blobs, chunks, torch, **kw):
    """Every way of calling: host blobs into host / device / no output; all OK, bytes and digests equal."""
    want = np.frombuffer(b"".join(sha(c) for c in chunks), np.uint8).reshape(-1, 32)
    lens = [len(c) for c in chunks]
    for out in ("host", "device", None):
        st, data, dig = eng.blob_decode_batch(blobs, lens, digests=want.tobytes(), out=out, **kw)
        assert (st == 0).all(), (out, st.tolist())
        assert (dig == want).all(), out
        if out is not None:
            for k, c in enumerate(chunks):
                got = data[k] if out == "host" else data[k].cpu().numpy().tobytes()
                assert got == c, (out, k)


ENCODERS = ("blob_encode_batch_z", "blob_encode_batch_lz", "blob_encode_batch_lze", "blob_encode_batch_lzh",
            "blob_encode_batch_lzl")


def test_round_trip_of_every_encoder_on_the_form_cases_from_host_and_device(eng, torch):
    parts = [p for p, _ in zf.form_cases()]
    chunks = [p.tobytes() for p in parts]
    buf, off, ln = pack(parts, 5)
    raw, boff, _ = eng.blob_encode_batch(buf, off, ln)
    blob_sets = {"raw": [raw[int(boff[i]):int(boff[i + 1])].tobytes() for i in range(len(parts))]}
    for name in ENCODERS:
        blob_sets[name] = getattr(eng, name)(buf, off, ln)[0]
    for name, blobs in blob_sets.items():
        check(eng, blobs, chunks, torch)
        # the same blobs at ragged offsets of a device buffer, into device output
        bb, bo, bl = pack([np.frombuffer(b, np.uint8) for b in blobs], 7)
        st, data, dig = eng.blob_decode_batch((to_dev(torch, bb), bo, bl), [len(c) for c in chunks], out="device")
        assert (st == 0).all(), name
        assert all(data[k].cpu().numpy().tobytes() == c for k, c in enumerate(chunks)), name


def test_round_trip_on_chunker_output_verify_only(eng, torch):
    img = np.concatenate([corpora(6 << 20, 3)["text"], np.zeros(1 << 20, np.uint8), corpora(5 << 20, 4)["binary"]])
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), d, [0], [len(img)])
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    for name in ENCODERS:
        blobs, _ = getattr(eng, name)(d, starts, ends - starts)
        st, data, dig = eng.blob_decode_batch(blobs, ends - starts, digests=rec["digest"].tobytes(), out=None)
        assert data is None and (st == 0).all(), name
        assert (dig == rec["digest"]).all(), name


def test_libzstd_frames_of_every_level_on_4_mib_chunks_and_one_16_mib_chunk(eng, torch):
    items = libzstd_payloads(4 << 20, 5)
    blobs = [zblob(p) for _, _, p, _ in items]
    chunks = [c for _, _, _, c in items]
    big = corpora(16 << 20, 6)["text"].tobytes()
    blobs.append(zblob(pa.Codec("zstd", compression_level=3).compress(big, asbytes=True)))
    chunks.append(big)
    check(eng, blobs, chunks, torch)


def test_fixture_frames(eng, torch):
    cases = zd.fixture_cases()
    check(eng, [zblob(p) for p, _ in cases.values()], [d for _, d in cases.values()], torch)


def test_index_end_to_end_verify_and_one_wrong_digest(eng, torch):
    img = np.concatenate([corpora(8 << 20, 7)["text"], corpora(4 << 20, 8)["binary"]])
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), d, [0], [len(img)])
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    blobs, _ = eng.blob_encode_batch_lzh(d, starts, ends - starts)
    ie, idg = eng.didx_parse(eng.didx_build(rec))
    clen = np.diff(np.concatenate([[0], ie])).astype(np.uint64)
    st, _, dig = eng.blob_decode_batch(blobs, clen, digests=idg.tobytes(), out=None)
    assert (st == _lib.DEC_OK).all() and (dig == idg).all()
    bad = idg.copy()
    bad[2, 5] ^= 1
    st, _, dig = eng.blob_decode_batch(blobs, clen, digests=bad.tobytes(), out=None)
    assert st[2] == _lib.DEC_BAD_DIGEST and (np.delete(st, 2) == _lib.DEC_OK).all()
    assert (dig == idg).all()


def test_per_blob_statuses(eng, torch):
    cases = zd.fixture_cases()
    ck_payload, ck_data = cases["checksum_raw"]
    text = corpora(300_000, 9)["text"].tobytes()
    good = zblob(pa.Codec("zstd", compression_level=3).compress(text, asbytes=True))
    # a byte inside checksum_raw's first Raw_Block, with the blob CRC fixed: only the content checksum sees it
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
    crc_flip = bytearray(good)
    crc_flip[40] ^= 1
    blobs = [good, b"\0" * 8 + good[8:], bytes(crc_flip), ENCRYPTED + good[8:], ENCR_COMPR + good[8:], good,
             zblob(bytes(flipped)), good[:7], zblob(b"\x28\xb5\x2f\xfd\x00")]
    lens = [len(text), len(text), len(text), len(text), len(text), len(text) + 1, len(ck_data), 0, 0]
    want = [_lib.DEC_OK, _lib.DEC_BAD_MAGIC, _lib.DEC_BAD_CRC, _lib.DEC_ENCRYPTED, _lib.DEC_ENCRYPTED, _lib.DEC_BAD_SIZE,
            _lib.DEC_BAD_CHECKSUM, _lib.DEC_BAD_MAGIC, _lib.DEC_BAD_FRAME]
    for out in ("host", None):
        st, data, _ = eng.blob_decode_batch(blobs, lens, out=out)
        assert st.tolist() == want, out
    # bad arguments
    L, h = eng._L, eng._h
    arr = np.frombuffer(good, np.uint8)
    o, l, cl = (np.array([x], np.uint64) for x in (0, len(good), len(text)))
    st = np.zeros(1, np.int32)
    args = [h, arr.ctypes.data, o.ctypes.data, l.ctypes.data, 1, cl.ctypes.data, None, None, None, st.ctypes.data, None]
    assert L.pbsgpu_blob_decode_batch(*args) == 0 and st[0] == 0
    for k in (0, 1, 2, 3, 5, 9):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_decode_batch(*bad) == _lib.EINVAL, k
    outb = np.zeros(len(text), np.uint8)
    bad = list(args)
    bad[7] = outb.ctypes.data          # out without out_off
    assert L.pbsgpu_blob_decode_batch(*bad) == _lib.EINVAL
    big = np.array([1 << 32], np.uint64)
    bad = list(args)
    bad[5] = big.ctypes.data
    assert L.pbsgpu_blob_decode_batch(*bad) == _lib.EINVAL
    assert L.pbsgpu_blob_decode_batch(h, None, None, None, 0, None, None, None, None, None, None) == 0


def libzstd_result(payload: bytes, size: int):
    """What upstream's streaming libzstd decoder reads from the payload, or None where it fails or reads another size."""
    got = zstd_stream_ref.stream_decode(payload)
    return got if isinstance(got, bytes) and len(got) == size else None


def test_corrupted_frames_never_pass_where_libzstd_fails(eng, torch):
    """Truncations at every block edge and seeded byte flips, the blob CRC recomputed, each between intact neighbours."""
    zstd_stream_ref.require()
    cases = zd.fixture_cases()
    text = corpora(400_000, 10)["text"].tobytes()
    srcs = [(cases[k][0], cases[k][1]) for k in ("small_window", "two_frames", "handmade", "nofcs")]
    srcs.append((pa.Codec("zstd", compression_level=19).compress(text, asbytes=True), text))
    rng = random.Random(13)
    bad_payloads = []
    for payload, data in srcs:
        edges, pos = [], 0
        for kind, fr in zd.split_payload(payload):
            if kind == "zstd":
                fhd = fr[4]
                p = 5 + (not (fhd >> 5) & 1) + (0, 1, 2, 4)[fhd & 3] + ((1 if (fhd >> 5) & 1 else 0), 2, 4, 8)[fhd >> 6]
                while True:
                    edges.append(pos + p)
                    h = int.from_bytes(fr[p:p + 3], "little")
                    p += 3 + (1 if (h >> 1) & 3 == 1 else h >> 3)
                    if h & 1:
                        break
            pos += len(fr)
        for e in edges[:40]:
            for cut in (e, e + 1, e + 3):
                bad_payloads.append((payload[:cut], data))
        for _ in range(60):
            b = bytearray(payload)
            for _ in range(rng.randint(1, 3)):
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            bad_payloads.append((bytes(b), data))
    neighbour = zblob(pa.Codec("zstd", compression_level=1).compress(text, asbytes=True))
    for lo in range(0, len(bad_payloads), 64):
        group = bad_payloads[lo:lo + 64]
        blobs, lens = [], []
        for payload, data in group:
            blobs += [neighbour, zblob(payload)]
            lens += [len(text), len(data)]
        blobs.append(neighbour)
        lens.append(len(text))
        st, out, _ = eng.blob_decode_batch(blobs, lens, out="host")
        assert (st[0::2] == _lib.DEC_OK).all()
        for k, (payload, data) in enumerate(group):
            ref = libzstd_result(payload, len(data))
            s = st[2 * k + 1]
            if ref is None:
                assert s != _lib.DEC_OK, (lo + k, s)
            if s == _lib.DEC_OK:
                assert out[2 * k + 1] == ref, lo + k


def test_a_4_gib_batch_crosses_the_pass_edges(eng, torch):
    """1 040 chunks of 4 MiB (4.06 GiB, more than two passes of ZDEC_PASS_BYTES), verify only, from a device base."""
    n, size = 1040, 4 << 20
    d = torch.empty(n * size, dtype=torch.uint8, device="cuda")
    eng.corpus_fill(pg.corpus(seed=21, file_len=size, run_blocks=4), 0, n, d, size)
    d.view(n, size)[::3, : 1 << 20] = 0                  # zero runs: every third blob is a zstd frame
    torch.cuda.synchronize()                             # torch's stream is not ordered with the engine's
    off = np.arange(n, dtype=np.uint64) * size
    ln = np.full(n, size, np.uint64)
    want = eng.sha256_batch(d, off, ln)
    # the blobs back to back in one host buffer, encoded a quarter at a time to bound host memory
    buf = np.zeros(n * (size + 12), np.uint8)
    boff, blen, pos = np.zeros(n, np.uint64), np.zeros(n, np.uint64), 0
    for g in range(0, n, n // 4):
        blobs, _ = eng.blob_encode_batch_z(d, off[g:g + n // 4], ln[g:g + n // 4])
        for k, b in enumerate(blobs):
            buf[pos:pos + len(b)] = np.frombuffer(b, np.uint8)
            boff[g + k], blen[g + k] = pos, len(b)
            pos += len(b)
        del blobs
    del d
    torch.cuda.empty_cache()
    assert (blen < size + 12).sum() >= n // 3
    st, data, dig = eng.blob_decode_batch((buf, boff, blen), ln, digests=want.tobytes(), out=None)
    assert data is None and (st == _lib.DEC_OK).all() and (dig == want).all()
