"""pbsgpu_blob_encode_batch_lz on the GPU (K8 + K9): bit-exact against tests/zstd_lz_ref.py (blob_encode_lz), decoded by
libzstd (pyarrow's codec), never larger than the _z blob of the same chunk, at small and multi-GiB batch sizes and
through the writer."""
import zlib

import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg
from oracle import pyref
import zstd_lz_ref as lzref
from pbs_plus_b200 import transfer
from pbs_plus_b200._lib import EINVAL

pytestmark = pytest.mark.gpu
B = pyref.ZFRAME_BLOCK
pa = pytest.importorskip("pyarrow")


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=n, dtype=np.uint8)


def to_dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def decode(frame: bytes, size: int) -> bytes:
    return pa.Codec("zstd").decompress(frame, decompressed_size=size).to_pybytes() if size else b""


def check_blob(blob: bytes, chunk: bytes, crc: int):
    assert int.from_bytes(blob[8:12], "little") == zlib.crc32(blob[12:]) == crc
    if blob[:8] == pyref.BLOB_MAGIC_COMPRESSED:
        assert len(blob) < 12 + len(chunk) and decode(blob[12:], len(chunk)) == chunk
    else:
        assert blob[:8] == pyref.BLOB_MAGIC_UNCOMPRESSED and blob[12:] == chunk


def mixed_parts():
    """The _z test's cases plus compressible ones: text, records, periodic data, a whole-block match, text around
    zero runs off the block grid."""
    text = lzref.text_corpus(3 << 20, 5)
    per = np.tile(rnd(37, 76), 10_000)
    return [np.zeros(4 << 20, np.uint8), rnd(1_000_000, 70),
            np.concatenate([rnd(B, 71), np.zeros(2 * B, np.uint8), rnd(5, 72)]),
            np.concatenate([rnd(1000, 73), np.zeros(3 * B, np.uint8), rnd(B - 1000 + 77, 74)]),
            np.full(B + 1, 7, np.uint8), np.full(20, 0x41, np.uint8), np.full(16, 0x41, np.uint8),
            np.zeros(0, np.uint8), rnd(1, 75),
            np.concatenate([np.zeros(B, np.uint8), np.ones(1, np.uint8), np.zeros(B - 1, np.uint8)]),
            text[:1 << 20], text[(1 << 20) + 3:(2 << 20) + B + 17], text[:300], text[:B - 1], text[:B + 1],
            per, np.tile(np.arange(4, dtype=np.uint8), B // 4 * 2),
            np.concatenate([text[:B + 999], np.zeros(2 * B, np.uint8), text[B:B + 5000], rnd(3000, 77)])]


def pack(parts, shift):
    offs, pos = [], shift
    for p in parts:
        offs.append(pos)
        pos += len(p) + 1                                    # ragged: every source misaligned differently
    buf = np.full(pos + 64, 0xEE, np.uint8)
    for p, o in zip(parts, offs):
        buf[o:o + len(p)] = p
    return buf, np.array(offs, np.uint64), np.array([len(p) for p in parts], np.uint64)


def test_blob_encode_batch_lz_equals_the_restatement_for_a_mixed_batch(eng, torch):
    parts = mixed_parts()
    want = [lzref.blob_encode_lz(p.tobytes()) for p in parts]
    buf, off, ln = pack(parts, 3)
    kinds = set()
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = eng.blob_encode_batch_lz(base, off, ln)
        zblobs, _ = eng.blob_encode_batch_z(base, off, ln)
        for i, (blob, p) in enumerate(zip(blobs, parts)):
            assert blob == want[i], (i, len(blob), len(want[i]))
            check_blob(blob, p.tobytes(), int(crc[i]))
            assert len(blob) <= len(zblobs[i])
            kinds.add(blob[:8] == pyref.BLOB_MAGIC_COMPRESSED and len(blob) < len(zblobs[i]))
    assert kinds == {True, False}


def test_blob_encode_batch_lz_on_chunker_output(eng, torch):
    """The NEW chunks of a text + zero-run + random image: every blob at most its _z blob, strictly smaller in total."""
    img = np.concatenate([lzref.text_corpus(6 << 20, 8), np.zeros(3 << 20, np.uint8), rnd(3 << 20, 81),
                          lzref.text_corpus(2 << 20, 9)])
    img[(7 << 20) + 4321:(7 << 20) + 9999] = 0
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), d, [0], [len(img)])
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    blobs, crc = eng.blob_encode_batch_lz(d, starts, ends - starts)
    zblobs, _ = eng.blob_encode_batch_z(d, starts, ends - starts)
    for k, (s0, e0) in enumerate(zip(starts, ends)):
        chunk = img[int(s0):int(e0)].tobytes()
        assert blobs[k] == lzref.blob_encode_lz(chunk)
        check_blob(blobs[k], chunk, int(crc[k]))
        assert len(blobs[k]) <= len(zblobs[k])
    total, ztotal = sum(map(len, blobs)), sum(map(len, zblobs))
    assert total < ztotal and total < 0.8 * len(img)


def test_blob_encode_batch_lz_large_device_batch(eng, torch):
    """4 GiB of 4 MiB chunks in device memory (several passes of the match stage): libzstd decodes every frame back to
    its chunk, and a seeded sample of chunks equals the restatement.  The image repeats a 64 MiB tile, so a chunk's blob must
    equal that of the same chunk in the first tile, which is decoded."""
    CH = 4 << 20
    tile = np.concatenate([lzref.text_corpus(40 << 20, 12), np.zeros(8 << 20, np.uint8), rnd(16 << 20, 13)])
    reps = (4 << 30) // len(tile)
    d = to_dev(torch, tile).repeat(reps)
    torch.cuda.synchronize()                                # the engine's streams do not wait for torch's
    n = len(d) // CH
    off = np.arange(n, dtype=np.uint64) * np.uint64(CH)
    ln = np.full(n, CH, np.uint64)
    blobs, crc = eng.blob_encode_batch_lz(d, off, ln)
    per_tile = len(tile) // CH
    for k in range(per_tile):
        check_blob(blobs[k], tile[k * CH:(k + 1) * CH].tobytes(), int(crc[k]))
    for k in range(per_tile, n):
        assert blobs[k] == blobs[k % per_tile] and crc[k] == crc[k % per_tile]
    for k in np.random.default_rng(14).choice(per_tile, 2, replace=False):
        s0 = int(k) * CH
        assert blobs[int(k)] == lzref.blob_encode_lz(tile[s0:s0 + CH].tobytes())
    assert sum(map(len, blobs)) < 0.7 * n * CH


def test_dedup_writer_uploads_lz_datablobs(eng, torch):
    blobs = []
    w = transfer.DedupWriter(eng, pg.make_config(1 << 16), eng.digest_set(), upload_blob=lambda d, b: blobs.append((d, b)),
                             blob_compression="lz")
    text = lzref.text_corpus(3_000_000, 20)
    sparse = text.copy()
    sparse[1_000_000:2_000_000] = 0
    files = [("notes.txt", text), ("disk.img", sparse), ("copy.txt", text.copy()), ("rand", rnd(200_000, 21))]
    for name, data in files:
        w.WriteEntry(transfer.Entry(name, len(data)), data.tobytes())
    w.Finish()
    ref = oracle.chunk_digest_streams(oracle.config(1 << 16), [d for _, d in files])
    want, seen, start = [], set(), {}
    for r in ref:
        i = int(r["stream"]); s0 = start.get(i, 0); e0 = int(r["end_off"]); start[i] = e0
        d = bytes(r["digest"])
        if d not in seen:
            seen.add(d)
            want.append((d, lzref.blob_encode_lz(files[i][1][s0:e0].tobytes())))
    assert blobs == want
    with pytest.raises(ValueError):
        transfer.DedupWriter(eng, pg.make_config(1 << 16), blob_compression="zstd")


def test_blob_encode_batch_lz_error_paths(eng, torch):
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
    assert L.pbsgpu_blob_encode_batch_lz(h, *args) == 0
    assert out[:8].tobytes() == pyref.BLOB_MAGIC_UNCOMPRESSED and int(ol[0]) == 112
    assert L.pbsgpu_blob_encode_batch_lz(None, *args) == EINVAL
    for k in (0, 1, 2, 4, 5, 6):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_encode_batch_lz(h, *bad) == EINVAL, k
    big = np.full(1, 1 << 40, np.uint64)
    assert L.pbsgpu_blob_encode_batch_lz(h, d.data_ptr(), p(off), p(big), 1, p(out), p(oo), p(ol), p(crc)) == EINVAL
    assert L.pbsgpu_blob_encode_batch_lz(h, None, None, None, 0, None, None, None, None) == 0
    blobs, crc = eng.blob_encode_batch_lz(d, [], [])
    assert blobs == [] and len(crc) == 0
