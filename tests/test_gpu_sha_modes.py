"""Every SHA-256 kernel instantiation against hashlib: each PBSGPU_SHA_MODE (throughput mixes 0/1/2/3/7, latency-only
10..14), through the throughput kernel alone (PBSGPU_SHA_HYBRID=0), the hybrid launch (=2, no SM partition) and the
long-chunk arena (early input release).  The inputs put every start offset mod 16 under the 16-byte vector loader,
lengths 0..200 and around multiples of 64 under the tail/padding path, and multi-MiB chunks under the latency kernel."""
import hashlib
import os

import numpy as np
import pytest

import pbs_plus_b200 as pg

pytestmark = pytest.mark.gpu

MODES = [0, 1, 2, 3, 7, 10, 11, 12, 13, 14]
PATHS = {"hybrid0": {"PBSGPU_SHA_HYBRID": "0", "PBSGPU_PARTITION_SMS": "0"},
         "hybrid2": {"PBSGPU_SHA_HYBRID": "2", "PBSGPU_PARTITION_SMS": "0"},
         "arena": {"PBSGPU_SHA_HYBRID": "2", "PBSGPU_PARTITION_SMS": "0"}}


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


def _engine(env):
    os.environ.update(env)
    try:
        return pg.Engine(0)
    finally:
        for k in env:
            del os.environ[k]


@pytest.fixture(scope="module")
def ranges():
    """(buffer, offsets, lengths): short and block-edge lengths at every offset mod 16, plus a few multi-MiB ranges"""
    rng = np.random.default_rng(11)
    lens = list(range(0, 201))
    lens += [64 * k + d for k in (4, 5, 16, 17, 63, 64, 1000) for d in (-9, -8, -1, 0, 1, 55, 56)]
    lens += [(3 << 20) + 5, (5 << 20) + 63, 8 << 20]
    offs, pos = [], 0
    for i, n in enumerate(lens):
        pos += i % 16 - pos % 16 + (16 if pos % 16 > i % 16 else 0)   # start offset = i mod 16
        offs.append(pos)
        pos += n
    buf = rng.integers(0, 256, size=pos + 64, dtype=np.uint8)
    return buf, np.array(offs, dtype=np.uint64), np.array(lens, dtype=np.uint64)


@pytest.fixture(scope="module")
def streams():
    """random streams with zero runs (cut at the maximum chunk size: the long class) at every start offset mod 16"""
    rng = np.random.default_rng(12)
    arrs = []
    for i in range(6):
        a = rng.integers(0, 256, size=5_000_000 + 4099 * i, dtype=np.uint8)
        if i % 2:
            a[1_000_000: 1_000_000 + 9_000_000 // 2] = 0
        arrs.append(a)
    arrs.append(rng.integers(0, 256, size=777, dtype=np.uint8))
    offs, pos = [], 0
    for i, a in enumerate(arrs):
        pos += 16 + (3 * i) % 16 - pos % 16
        offs.append(pos)
        pos += len(a)
    buf = np.zeros(pos + 64, dtype=np.uint8)
    for a, o in zip(arrs, offs):
        buf[o:o + len(a)] = a
    return buf, np.array(offs, dtype=np.uint64), np.array([len(a) for a in arrs], dtype=np.uint64)


def _check_records(rec, buf, off, ln):
    assert len(rec) > 0
    start = {}
    for r in rec:
        s, end = int(r["stream"]), int(r["end_off"])
        lo = start.get(s, 0)
        data = buf[int(off[s]) + lo: int(off[s]) + end]
        assert bytes(r["digest"]) == hashlib.sha256(data.tobytes()).digest(), (s, lo, end)
        start[s] = end
    assert all(start[s] == int(ln[s]) for s in range(len(ln)) if ln[s])


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", MODES)
def test_sha_mode_digests_equal_hashlib(torch, ranges, streams, mode, path):
    e = _engine({"PBSGPU_SHA_MODE": str(mode), **PATHS[path]})
    try:
        buf, off, ln = ranges
        got = e.sha256_batch(torch.from_numpy(buf).cuda(), off, ln)
        for i in range(len(off)):
            want = hashlib.sha256(buf[int(off[i]): int(off[i]) + int(ln[i])].tobytes()).digest()
            assert got[i].tobytes() == want, (i, int(off[i]) % 16, int(ln[i]))

        sbuf, soff, sln = streams
        cfg = pg.make_config(1 << 20)
        assert int(cfg.max) >= 2 << 20   # the zero runs give multi-MiB chunks
        d = torch.from_numpy(sbuf).cuda()
        if path == "arena":
            job = e.submit(cfg, d, soff, sln, early_input=True)
            job.wait_input()
            rec, _ = job.wait()
        else:
            rec = e.chunk_digest_batch(cfg, d, soff, sln)
        _check_records(rec, sbuf, soff, sln)
        assert (np.diff(rec["end_off"].astype(np.int64))[np.diff(rec["stream"].astype(np.int64)) == 0] >= 2 << 20).any()
    finally:
        e.close()
