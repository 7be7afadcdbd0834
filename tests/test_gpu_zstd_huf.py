"""pbsgpu_blob_encode_batch_lzh on the GPU (K8 + K9 + K10 with its full-alphabet flag): bit-exact against
tests/zstd_huf_ref.py (blob_encode_lzh), decoded by libzstd (pyarrow's codec), never larger than the _lze blob of the same
chunk, at small and multi-GiB batch sizes, through the writer and through the stream's blob mode."""
import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg
from oracle import pyref
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from pbs_plus_b200 import transfer
from pbs_plus_b200._lib import EINVAL
from test_gpu_round2 import _payload_stream
from test_gpu_stream_blobs import engine, write_stream
from test_gpu_zstd_ent import entropy_parts
from test_gpu_zstd_lz import check_blob, mixed_parts, pack, rnd, to_dev

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


def binary_parts():
    """Blocks that take each tree form of the full-alphabet literals: the binary corpus at ragged lengths, largest
    literal 129 / 200 / 255 in text, two distinct weights over a sparse alphabet (weight 0 holds most states), odd and
    even weight counts, a uniform 256-value histogram (no tree form: raw), and a small dense alphabet (direct form)."""
    binary = hufref.binary_corpus(3 * B + 777, 50)
    out = [binary, binary[:5000], binary[:B + 1]]
    for top in (129, 200, 255):
        t = lzref.text_corpus(30000, top).copy()
        t[::991] = top
        out.append(t)
    out.append(np.random.default_rng(51).choice(np.array([5, 200], np.uint8), 20000))
    for top in (130, 131):
        p = 1.0 / np.arange(1, top + 2)
        out.append(np.random.default_rng(top).choice(top + 1, 40000, p=p / p.sum()).astype(np.uint8))
    out.append(np.tile(np.arange(256, dtype=np.uint8), 200))
    p = np.array([20, 14, 12, 10, 9, 8, 7, 6, 5, 4, 3, 2], float)
    out.append(np.random.default_rng(52).choice(12, 50000, p=p / p.sum()).astype(np.uint8))
    return out


def test_blob_encode_batch_lzh_equals_the_restatement_for_a_mixed_batch(eng, torch):
    parts = mixed_parts() + entropy_parts() + binary_parts()
    want = [hufref.blob_encode_lzh(p.tobytes()) for p in parts]
    buf, off, ln = pack(parts, 7)
    smaller = set()
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = eng.blob_encode_batch_lzh(base, off, ln)
        lzeblobs, _ = eng.blob_encode_batch_lze(base, off, ln)
        for i, (blob, p) in enumerate(zip(blobs, parts)):
            assert blob == want[i], (i, len(blob), len(want[i]))
            check_blob(blob, p.tobytes(), int(crc[i]))
            assert len(blob) <= len(lzeblobs[i])
            smaller.add(len(blob) < len(lzeblobs[i]))
    assert smaller == {True, False}


def test_blob_encode_batch_lzh_on_chunker_output(eng, torch):
    """The NEW chunks of a binary + text + zero-run image: byte-exact, every blob at most its _lze blob, strictly
    smaller in total."""
    img = np.concatenate([hufref.binary_corpus(6 << 20, 8), lzref.text_corpus(2 << 20, 9), np.zeros(3 << 20, np.uint8),
                          hufref.binary_corpus(2 << 20, 10)])
    img[(7 << 20) + 4321:(7 << 20) + 9999] = 0
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), d, [0], [len(img)])
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    blobs, crc = eng.blob_encode_batch_lzh(d, starts, ends - starts)
    lzeblobs, _ = eng.blob_encode_batch_lze(d, starts, ends - starts)
    for k, (s0, e0) in enumerate(zip(starts, ends)):
        chunk = img[int(s0):int(e0)].tobytes()
        assert blobs[k] == hufref.blob_encode_lzh(chunk)
        check_blob(blobs[k], chunk, int(crc[k]))
        assert len(blobs[k]) <= len(lzeblobs[k])
    assert sum(map(len, blobs)) < sum(map(len, lzeblobs))


def test_blob_encode_batch_lzh_large_device_batch(eng, torch):
    """4 GiB of 4 MiB chunks in device memory (several passes of K9 / K10): libzstd decodes every frame of the first
    64 MiB tile back to its chunk, later tiles repeat those blobs, and a seeded sample equals the restatement."""
    CH = 4 << 20
    tile = np.concatenate([hufref.binary_corpus(24 << 20, 12), lzref.text_corpus(16 << 20, 13),
                           np.zeros(8 << 20, np.uint8), rnd(16 << 20, 14)])
    reps = (4 << 30) // len(tile)
    d = to_dev(torch, tile).repeat(reps)
    torch.cuda.synchronize()                                # the engine's streams do not wait for torch's
    n = len(d) // CH
    off = np.arange(n, dtype=np.uint64) * np.uint64(CH)
    ln = np.full(n, CH, np.uint64)
    blobs, crc = eng.blob_encode_batch_lzh(d, off, ln)
    per_tile = len(tile) // CH
    for k in range(per_tile):
        check_blob(blobs[k], tile[k * CH:(k + 1) * CH].tobytes(), int(crc[k]))
    for k in range(per_tile, n):
        assert blobs[k] == blobs[k % per_tile] and crc[k] == crc[k % per_tile]
    for k in np.random.default_rng(15).choice(10, 2, replace=False):   # two of the binary and text chunks
        s0 = int(k) * CH
        assert blobs[int(k)] == hufref.blob_encode_lzh(tile[s0:s0 + CH].tobytes())


def test_dedup_writer_uploads_lzh_datablobs(eng, torch):
    blobs = []
    w = transfer.DedupWriter(eng, pg.make_config(1 << 16), eng.digest_set(), upload_blob=lambda d, b: blobs.append((d, b)),
                             blob_compression="lzh")
    binary = hufref.binary_corpus(2_000_000, 20)
    sparse = binary.copy()
    sparse[500_000:1_500_000] = 0
    files = [("app.bin", binary), ("disk.img", sparse), ("copy.bin", binary.copy()), ("rand", rnd(200_000, 21)),
             ("notes.txt", lzref.text_corpus(700_000, 22))]
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
            want.append((d, hufref.blob_encode_lzh(files[i][1][s0:e0].tobytes())))
    assert blobs == want


def test_stream_blob_mode_lzh_equals_the_batch_call():
    """64 KiB windows, so window ends fall inside the files and inside chunks: the stream's blobs equal the batch call's
    and the restatement's."""
    e = engine(1 << 16)
    try:
        files = [hufref.binary_corpus(900_000, 30), np.zeros(200_000, np.uint8), lzref.text_corpus(350_001, 31),
                 hufref.binary_corpus(190_000, 32)]
        stream, starts = _payload_stream(files)
        avg = 1 << 16
        ref = oracle.chunk_digest_forced(oracle.config(avg), stream, np.array(starts, np.uint64))
        ends = ref["end_off"].astype(np.uint64)
        off = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
        want, _ = e.blob_encode_batch_lzh(stream, off, ends - off)
        st = e.stream(pg.make_config(avg))
        st.blob_mode("lzh")
        rec, blobs = write_stream(st, files, 50_001, True)
        st.close()
        assert rec["end_off"].tolist() == ref["end_off"].tolist()
        assert blobs == want
        for b, o, l in list(zip(blobs, off, ends - off))[::5]:
            assert b == hufref.blob_encode_lzh(stream[int(o):int(o + l)].tobytes())
    finally:
        e.close()


def test_blob_encode_batch_lzh_error_paths(eng, torch):
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
    assert L.pbsgpu_blob_encode_batch_lzh(h, *args) == 0
    assert out[:8].tobytes() == pyref.BLOB_MAGIC_UNCOMPRESSED and int(ol[0]) == 112
    assert L.pbsgpu_blob_encode_batch_lzh(None, *args) == EINVAL
    for k in (0, 1, 2, 4, 5, 6):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_encode_batch_lzh(h, *bad) == EINVAL, k
    big = np.full(1, 1 << 40, np.uint64)
    assert L.pbsgpu_blob_encode_batch_lzh(h, d.data_ptr(), p(off), p(big), 1, p(out), p(oo), p(ol), p(crc)) == EINVAL
    assert L.pbsgpu_blob_encode_batch_lzh(h, None, None, None, 0, None, None, None, None) == 0
    blobs, crc = eng.blob_encode_batch_lzh(d, [], [])
    assert blobs == [] and len(crc) == 0
    with pytest.raises(ValueError):
        transfer.DedupWriter(eng, pg.make_config(1 << 16), blob_compression="lzx")
