"""pbsgpu_blob_encode_batch_lze on the GPU (K8 + K9 + K10): bit-exact against tests/zstd_ent_ref.py (blob_encode_lze),
decoded by libzstd (pyarrow's codec), never larger than the _lz blob of the same chunk, at small and multi-GiB batch
sizes and through the writer."""
import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg
from oracle import pyref
import zstd_ent_ref as entref
import zstd_lz_ref as lzref
from pbs_plus_b200 import transfer
from pbs_plus_b200._lib import EINVAL
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


def entropy_parts():
    """Blocks that take each literal and table form of K10: one literal value, two values, largest value 128 (Huffman)
    and 129 (raw), literal counts at the one / four stream boundary, RLE-mode columns and a single sequence."""
    text = lzref.text_corpus(B, 40)
    two = np.random.default_rng(41).choice(np.array([97, 98], np.uint8), 20000)
    per = np.tile(np.frombuffer(b"abcdefgh", np.uint8), 4000)
    hi = np.frombuffer(bytes(lzref.text_corpus(30000, 42)), np.uint8).copy()
    hi[::997] = 128
    hi129 = hi.copy()
    hi129[5] = 129
    out = [two, per, hi, hi129, np.concatenate([np.full(300, 7, np.uint8), rnd(300, 43), rnd(300, 43)])]
    for nl in (1023, 1024):
        lits = np.random.default_rng(nl).choice(np.frombuffer(b"etaoin shr", np.uint8), nl)
        out.append(np.concatenate([lits, np.tile(lits[:64], 40)]))
    return out + [text[:5000], text]


def test_blob_encode_batch_lze_equals_the_restatement_for_a_mixed_batch(eng, torch):
    parts = mixed_parts() + entropy_parts()
    want = [entref.blob_encode_lze(p.tobytes()) for p in parts]
    buf, off, ln = pack(parts, 5)
    kinds = set()
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = eng.blob_encode_batch_lze(base, off, ln)
        lzblobs, _ = eng.blob_encode_batch_lz(base, off, ln)
        for i, (blob, p) in enumerate(zip(blobs, parts)):
            assert blob == want[i], (i, len(blob), len(want[i]))
            check_blob(blob, p.tobytes(), int(crc[i]))
            assert len(blob) <= len(lzblobs[i])
            kinds.add(blob[:8] == pyref.BLOB_MAGIC_COMPRESSED and len(blob) < len(lzblobs[i]))
    assert kinds == {True, False}


def test_blob_encode_batch_lze_on_chunker_output(eng, torch):
    """The NEW chunks of a text + zero-run + random image: every blob at most its _lz blob, strictly smaller in total."""
    img = np.concatenate([lzref.text_corpus(6 << 20, 8), np.zeros(3 << 20, np.uint8), rnd(3 << 20, 81),
                          lzref.text_corpus(2 << 20, 9)])
    img[(7 << 20) + 4321:(7 << 20) + 9999] = 0
    d = to_dev(torch, img)
    rec = eng.chunk_digest_batch(pg.make_config(1 << 20), d, [0], [len(img)])
    ends = rec["end_off"].astype(np.uint64)
    starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
    blobs, crc = eng.blob_encode_batch_lze(d, starts, ends - starts)
    lzblobs, _ = eng.blob_encode_batch_lz(d, starts, ends - starts)
    for k, (s0, e0) in enumerate(zip(starts, ends)):
        chunk = img[int(s0):int(e0)].tobytes()
        assert blobs[k] == entref.blob_encode_lze(chunk)
        check_blob(blobs[k], chunk, int(crc[k]))
        assert len(blobs[k]) <= len(lzblobs[k])
    total, lztotal = sum(map(len, blobs)), sum(map(len, lzblobs))
    assert total < 0.85 * lztotal


def test_blob_encode_batch_lze_large_device_batch(eng, torch):
    """4 GiB of 4 MiB chunks in device memory (several passes of K9 / K10): libzstd decodes every frame of the first
    64 MiB tile back to its chunk, later tiles repeat those blobs, and a seeded sample equals the restatement."""
    CH = 4 << 20
    tile = np.concatenate([lzref.text_corpus(40 << 20, 12), np.zeros(8 << 20, np.uint8), rnd(16 << 20, 13)])
    reps = (4 << 30) // len(tile)
    d = to_dev(torch, tile).repeat(reps)
    torch.cuda.synchronize()                                # the engine's streams do not wait for torch's
    n = len(d) // CH
    off = np.arange(n, dtype=np.uint64) * np.uint64(CH)
    ln = np.full(n, CH, np.uint64)
    blobs, crc = eng.blob_encode_batch_lze(d, off, ln)
    per_tile = len(tile) // CH
    for k in range(per_tile):
        check_blob(blobs[k], tile[k * CH:(k + 1) * CH].tobytes(), int(crc[k]))
    for k in range(per_tile, n):
        assert blobs[k] == blobs[k % per_tile] and crc[k] == crc[k % per_tile]
    for k in np.random.default_rng(14).choice(10, 2, replace=False):   # two of the text chunks
        s0 = int(k) * CH
        assert blobs[int(k)] == entref.blob_encode_lze(tile[s0:s0 + CH].tobytes())
    assert sum(map(len, blobs)) < 0.52 * n * CH


def test_dedup_writer_uploads_lze_datablobs(eng, torch):
    blobs = []
    w = transfer.DedupWriter(eng, pg.make_config(1 << 16), eng.digest_set(), upload_blob=lambda d, b: blobs.append((d, b)),
                             blob_compression="lze")
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
            want.append((d, entref.blob_encode_lze(files[i][1][s0:e0].tobytes())))
    assert blobs == want


def test_blob_encode_batch_lze_error_paths(eng, torch):
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
    assert L.pbsgpu_blob_encode_batch_lze(h, *args) == 0
    assert out[:8].tobytes() == pyref.BLOB_MAGIC_UNCOMPRESSED and int(ol[0]) == 112
    assert L.pbsgpu_blob_encode_batch_lze(None, *args) == EINVAL
    for k in (0, 1, 2, 4, 5, 6):
        bad = list(args)
        bad[k] = None
        assert L.pbsgpu_blob_encode_batch_lze(h, *bad) == EINVAL, k
    big = np.full(1, 1 << 40, np.uint64)
    assert L.pbsgpu_blob_encode_batch_lze(h, d.data_ptr(), p(off), p(big), 1, p(out), p(oo), p(ol), p(crc)) == EINVAL
    assert L.pbsgpu_blob_encode_batch_lze(h, None, None, None, 0, None, None, None, None) == 0
    blobs, crc = eng.blob_encode_batch_lze(d, [], [])
    assert blobs == [] and len(crc) == 0
