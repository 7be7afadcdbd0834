"""K13 on the edge frames of tests/zstd_edge_frames.py, through pbsgpu_blob_decode_batch and _enc: every case in
batches with an intact libzstd blob between every two cases, from host and ragged device bases, into host output,
device output at every out_off residue mod 8, and no output.  Valid cases decode to their bytes and SHA-256, invalid
ones give their exact status, and the neighbours decode unchanged.  The encrypted run sends the same payloads through
the decryption stage; a host `out` gets no byte of an encrypted blob whose frame is refused."""
import random
import zlib

import numpy as np
import pytest

import crypt_ref
import zstd_edge_frames as ef
from pbs_plus_b200 import _lib
from pbs_plus_b200.engine import _ptr
from test_gpu_blob_decode import sha, zblob
from test_gpu_zstd_lz import pack, to_dev
from test_zstd_decode_cpu import corpora

pytestmark = pytest.mark.gpu
pa = pytest.importorskip("pyarrow")
KEY = bytes(range(7, 39))
SENTINEL = 0xA5


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
    import pbs_plus_b200 as pg
    e = pg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def batch():
    """(blobs' payloads, chunk_len, content or None, status) with a libzstd neighbour before, between and after the cases"""
    text = corpora(70_000, 31)["text"].tobytes()
    nb = pa.Codec("zstd", compression_level=3).compress(text, asbytes=True)
    items = [(nb, len(text), text, _lib.DEC_OK)]
    for c in ef.edge_cases():
        items += [(c.payload, c.size, c.content, c.status), (nb, len(text), text, _lib.DEC_OK)]
    return items


def expect(items, st, chunks, where):
    for k, (_, size, content, want) in enumerate(items):
        name = "neighbour" if k % 2 == 0 else ef.edge_cases()[k // 2].name
        assert st[k] == want, (where, name, int(st[k]), want)
        if content is not None and chunks is not None:
            assert chunks[k] == content, (where, name)


def raw_call(eng, fn_args, blobs, lens, out, ooff):
    """pbsgpu_blob_decode_batch(_enc) with the caller's own `out` and out_off."""
    L = eng._L
    base = np.frombuffer(b"".join(blobs), np.uint8)
    o = np.zeros(len(blobs), np.uint64)
    o[1:] = np.cumsum([len(b) for b in blobs])[:-1]
    l = np.array([len(b) for b in blobs], np.uint64)
    cl = np.array(lens, np.uint64)
    st = np.zeros(len(blobs), np.int32)
    fn = L.pbsgpu_blob_decode_batch_enc if fn_args else L.pbsgpu_blob_decode_batch
    rc = fn(eng._h, *fn_args, base.ctypes.data, o.ctypes.data, l.ctypes.data, len(blobs), cl.ctypes.data, None,
            _ptr(out), ooff.ctypes.data, st.ctypes.data, None)
    assert rc == 0
    return st


def residue_offsets(lens):
    """out_off of each chunk: 8-byte aligned starts plus k mod 8, so every residue is met"""
    ooff, pos = np.zeros(len(lens), np.uint64), 0
    for k, n in enumerate(lens):
        pos = (pos + 7) // 8 * 8 + k % 8
        ooff[k] = pos
        pos += n
    return ooff, pos + 8


def test_every_edge_case_between_intact_neighbours(eng, torch, batch):
    blobs = [zblob(p) for p, _, _, _ in batch]
    lens = [n for _, n, _, _ in batch]
    want = np.frombuffer(b"".join(sha(c) if c is not None else bytes(32) for _, _, c, _ in batch), np.uint8)
    want = want.reshape(-1, 32)
    bb, bo, bl = pack([np.frombuffer(b, np.uint8) for b in blobs], 7)
    for src_name, src in (("host", blobs), ("device", (to_dev(torch, bb), bo, bl))):
        for out in ("host", "device", None):
            st, data, dig = eng.blob_decode_batch(src, lens, digests=want.tobytes(), out=out)
            chunks = None if data is None else [d if d is None or out == "host" else d.cpu().numpy().tobytes()
                                                for d in data]
            expect(batch, st, chunks, (src_name, out))
            ok = st == _lib.DEC_OK
            assert (dig[ok] == want[ok]).all(), (src_name, out)
    # device output at every residue mod 8, the bytes around each chunk untouched
    ooff, total = residue_offsets(lens)
    dev = torch.full((total,), SENTINEL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    st = raw_call(eng, (), blobs, lens, dev, ooff)
    got = dev.cpu().numpy()
    expect(batch, st, None, "device residues")
    mask = np.ones(total, bool)
    for k, (_, n, content, _) in enumerate(batch):
        if content is not None:
            assert got[int(ooff[k]): int(ooff[k]) + n].tobytes() == content, k
        mask[int(ooff[k]): int(ooff[k]) + n] = False
    assert (got[mask] == SENTINEL).all()


def test_every_edge_case_through_the_decryption_stage(eng, torch, batch):
    rng = random.Random(41)

    def enc(payload):
        ct, tag = crypt_ref.gcm_encrypt(KEY, iv := rng.randbytes(16), payload)
        return crypt_ref.ENCR_COMPR_BLOB_MAGIC_1_0 + zlib.crc32(ct).to_bytes(4, "little") + iv + tag + ct

    blobs = [enc(p) for p, _, _, _ in batch]
    lens = [n for _, n, _, _ in batch]
    ident = crypt_ref.id_key(KEY)
    want = np.frombuffer(b"".join(crypt_ref.compute_digest(c, ident) if c is not None else bytes(32)
                                  for _, _, c, _ in batch), np.uint8).reshape(-1, 32)
    crypt = eng.crypt(KEY)
    try:
        st, data, dig = eng.blob_decode_batch_enc(crypt, blobs, lens, digests=want.tobytes(), out="host")
        expect(batch, st, data, "encrypted")
        ok = st == _lib.DEC_OK
        assert (dig[ok] == want[ok]).all()
        # a host `out` gets no byte of a blob whose frame is refused
        ooff, total = residue_offsets(lens)
        host = np.full(total, SENTINEL, np.uint8)
        st = raw_call(eng, (crypt._h,), blobs, lens, host, ooff)
        expect(batch, st, None, "encrypted, caller's out")
        for k, (_, n, content, _) in enumerate(batch):
            region = host[int(ooff[k]): int(ooff[k]) + n]
            if content is None:
                assert (region == SENTINEL).all(), ef.edge_cases()[k // 2].name
            else:
                assert region.tobytes() == content, k
    finally:
        crypt.close()
