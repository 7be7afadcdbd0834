"""The K3 matrix (tests/sha_matrix.py) on the GPU: every SHA-256 kernel instantiation, plain and keyed, against hashlib.

- the blocking byte-range calls with the throughput kernel and the simple variant, over the padding edges and
  multi-MiB ranges, from a host base and a ragged device base;
- the batch job on every launch path: the cuts equal the oracle's and the digests are hashlib's of those cuts, for the
  chunker (blocking call and early-input-release job) and for fixed-size cuts;
- the latency kernel over the padding edges and past 2^32 bits, each range a stream of one chunk in its head;
- the blocking decode of encrypted DataBlobs, whose keyed digest check is the other caller of the blocking launch;
- messages of 512 MiB and more, whose bit length needs the high length word, and the refusal of a 4 GiB range."""
import os

import numpy as np
import pytest

import sha_matrix as M
import pbs_plus_b200 as pg
from pbs_plus_b200 import _lib

pytestmark = pytest.mark.gpu
FIXED = 1 << 18


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


def engine(env):
    """A context opened with `env` added to the environment (the knobs are read once, at open)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return pg.Engine(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def ragged(torch, buf, shift: int = 5):
    """`buf` on the device at an odd distance from the allocation: (tensor to keep alive, base address)"""
    d = torch.zeros(len(buf) + shift, dtype=torch.uint8, device="cuda")
    d[shift:] = torch.from_numpy(buf).cuda()
    torch.cuda.synchronize()
    return d, d.data_ptr() + shift


def expected(buf, off, ln, keyed):
    return [M.digest(buf[int(o): int(o) + int(n)], keyed) for o, n in zip(off, ln)]


@pytest.fixture(scope="module")
def ranges():
    buf, off, ln = M.edges_and_long()
    return buf, off, ln, expected(buf, off, ln, False), expected(buf, off, ln, True)


# ---- blocking calls ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", list(M.KERNELS))
def test_blocking_digests_equal_hashlib(torch, ranges, kernel):
    buf, off, ln, plain, keyed = ranges
    e = engine(M.KERNELS[kernel])
    try:
        c = e.crypt(M.KEY)
        keep, dbase = ragged(torch, buf)
        for base in (buf, dbase):
            for want, got in ((plain, e.sha256_batch(base, off, ln)), (keyed, e.sha256_keyed_batch(c, base, off, ln))):
                bad = [(i, int(off[i]) % 16, int(ln[i])) for i in range(len(off)) if got[i].tobytes() != want[i]]
                assert not bad, (kernel, want is keyed, isinstance(base, int), bad[:8], len(bad))
        c.close()
    finally:
        e.close()


# ---- the batch job ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def streams():
    import oracle
    (buf, off, ln), parts = M.pack_streams(M.stream_parts())
    cuts = oracle.chunk_digest_streams(oracle.config(M.AVG), parts)
    fixed = np.zeros(len(M.fixed_cuts(parts, FIXED)), dtype=cuts.dtype)
    for r, (s, end) in zip(fixed, M.fixed_cuts(parts, FIXED)):
        r["stream"], r["end_off"] = s, end
    return buf, off, ln, {"chunker": cuts, "fixed": fixed}, {
        (kind, keyed): M.records(c, parts, keyed) for kind, c in (("chunker", cuts), ("fixed", fixed)) for keyed in (False, True)}


def check(got, cuts, want, what):
    assert len(got) == len(cuts), what
    assert (got["stream"] == cuts["stream"]).all() and (got["end_off"] == cuts["end_off"]).all(), what
    bad = [i for i in range(len(got)) if got["digest"][i].tobytes() != want["digest"][i].tobytes()]
    assert not bad, (what, bad[:8], len(bad))
    assert got.tobytes() == want.tobytes(), what


@pytest.mark.parametrize("path", list(M.PATHS))
def test_job_paths_give_hashlib_digests_at_the_oracle_cuts(torch, streams, path):
    buf, off, ln, cuts, want = streams
    e = engine(M.PATHS[path])
    try:
        c = e.crypt(M.KEY)
        cfg = pg.make_config(M.AVG)
        dev = torch.from_numpy(buf).cuda()
        got = {}
        for keyed in (False, True):
            crypt = c if keyed else None
            w = want["chunker", keyed]
            for base in (buf, dev):
                got[keyed] = e.chunk_digest_batch(cfg, base, off, ln, crypt=crypt)
                check(got[keyed], cuts["chunker"], w, (path, keyed, "batch", isinstance(base, np.ndarray)))
            job = e.submit(cfg, dev, off, ln, early_input=True, crypt=crypt)
            job.wait_input()
            check(job.wait()[0], cuts["chunker"], w, (path, keyed, "arena"))
            check(e.chunk_digest_batch(None, dev, off, ln, crypt=crypt, fixed_size=FIXED), cuts["fixed"],
                  want["fixed", keyed], (path, keyed, "fixed"))
        assert not {d.tobytes() for d in got[False]["digest"]} & {d.tobytes() for d in got[True]["digest"]}
        c.close()
    finally:
        e.close()


# ---- the latency kernel at the padding edges and past 2^32 bits: one chunk per stream, every chunk in the head -----
def one_chunk_each(rec, lens, streams, keyed, what):
    """rec has one chunk per non-empty stream, the whole stream, with hashlib's digest of it"""
    nz = [s for s, n in enumerate(lens) if n]
    assert rec["stream"].tolist() == nz and rec["end_off"].tolist() == [lens[s] for s in nz], what
    bad = [s for s, d in zip(nz, rec["digest"]) if d.tobytes() != M.digest(streams(s), keyed)]
    assert not bad, (what, bad[:8], len(bad))


@pytest.mark.parametrize("path", ["split_every_chunk", "split_every_chunk_partitioned"])
def test_split_kernel_digests_at_the_padding_edges(torch, path):
    buf, off, ln = M.edges()
    lens = [int(n) for n in ln]
    e = engine(M.PATHS[path])
    try:
        c = e.crypt(M.KEY)
        cfg = pg.make_config(M.EDGE_AVG)
        for keyed in (False, True):
            rec = e.chunk_digest_batch(cfg, buf, off, ln, crypt=c if keyed else None)
            one_chunk_each(rec, lens, lambda s: buf[int(off[s]): int(off[s]) + lens[s]], keyed, (path, "edges", keyed))
        c.close()
    finally:
        e.close()


@pytest.mark.parametrize("path", ["split_every_chunk", "split_every_chunk_partitioned"])
def test_split_kernel_digests_past_2_pow_32_bits(torch, path):
    lens = M.LONG_ZERO
    off = np.cumsum([0] + lens[:-1]).astype(np.uint64) + np.arange(len(lens), dtype=np.uint64) * 7 + 3
    dev = torch.zeros(int(off[-1]) + lens[-1] + 64, dtype=torch.uint8, device="cuda")
    e = engine(M.PATHS[path])
    try:
        c = e.crypt(M.KEY)
        cfg = pg.make_config(M.LONG_AVG)
        for keyed in (False, True):
            rec = e.chunk_digest_batch(cfg, dev, off, np.array(lens, np.uint64), crypt=c if keyed else None)
            one_chunk_each(rec, lens, lambda s: np.zeros(lens[s], np.uint8), keyed, (path, "zeros", keyed))
        c.close()
    finally:
        e.close()
        del dev


# ---- the decode of encrypted DataBlobs: the other caller of the blocking launch ---------------------------------
@pytest.fixture(scope="module")
def enc_blobs():
    buf, off, ln = M.edges()
    e = pg.Engine(0)
    try:
        c = e.crypt(M.KEY)
        iv = np.random.default_rng(41).integers(0, 256, size=16 * len(off), dtype=np.uint8).tobytes()
        blobs, _ = e.blob_encode_batch_enc(c, "raw", buf, off, ln, iv)
        c.close()
    finally:
        e.close()
    return blobs, ln, b"".join(expected(buf, off, ln, True))


@pytest.mark.parametrize("kernel", list(M.KERNELS))
def test_encrypted_blob_decode_checks_keyed_digests(enc_blobs, kernel):
    blobs, ln, keyed = enc_blobs
    e = engine(M.KERNELS[kernel])
    try:
        c = e.crypt(M.KEY)
        st, _, dig = e.blob_decode_batch_enc(c, blobs, ln, keyed, out=None)
        assert (st == _lib.DEC_OK).all(), (kernel, np.flatnonzero(st != _lib.DEC_OK)[:8])
        assert dig.tobytes() == keyed
        for i in (0, 345, len(blobs) - 1):   # empty, 44 bytes (keyed: two final blocks), 64000 + 63
            bad = bytearray(keyed)
            bad[32 * i + 31] ^= 1
            st, _, _ = e.blob_decode_batch_enc(c, blobs, ln, bytes(bad), out=None)
            assert st[i] == _lib.DEC_BAD_DIGEST and (np.delete(st, i) == _lib.DEC_OK).all(), (kernel, i)
        c.close()
    finally:
        e.close()


# ---- long messages: the high word of the bit length ---------------------------------------------------------------
LONG = [(1 << 29) - 1, 1 << 29, (1 << 29) + 37, (1 << 29) - 20]   # plain bits below, at, above 2^32; keyed above


@pytest.fixture(scope="module")
def long_ranges(torch):
    off, pos = [], 0
    for i, n in enumerate(LONG):
        pos += 1 + (2 * i + 1 - pos - 1) % 16   # odd device offsets: residues 1, 3, 5, 7 mod 16
        off.append(pos)
        pos += n
    host = np.frombuffer(np.random.default_rng(51).bytes(pos + 64), np.uint8)
    off, ln = np.array(off, np.uint64), np.array(LONG, np.uint64)
    dev = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    yield dev, off, ln, expected(host, off, ln, False), expected(host, off, ln, True)
    del dev


@pytest.mark.parametrize("kernel", list(M.KERNELS))
def test_messages_past_2_pow_32_bits(long_ranges, kernel):
    dev, off, ln, plain, keyed = long_ranges
    e = engine(M.KERNELS[kernel])
    try:
        c = e.crypt(M.KEY)
        got = e.sha256_batch(dev, off, ln)
        assert [g.tobytes() for g in got] == plain, kernel
        got = e.sha256_keyed_batch(c, dev, off, ln)
        assert [g.tobytes() for g in got] == keyed, kernel
        for call in (lambda o, l: e.sha256_batch(dev, o, l), lambda o, l: e.sha256_keyed_batch(c, dev, o, l)):
            with pytest.raises(pg.PbsGpuError) as err:
                call([0, 1], [5, 1 << 32])
            assert err.value.code == _lib.EINVAL
        c.close()
    finally:
        e.close()
