"""pbsgpu_deflate_batch on the GPU (K9a's Deflate parse + K15): byte-identical to tests/deflate_ref.py on every CPU
case, from host and ragged device bases into host and device out; pieces joined through `more` and the EINVAL of an
unaligned piece; CRCs against zlib; out_len <= bound on random data; 256 MiB of each corpus inflates through zlib; and
one call that crosses a pass edge."""
import zlib

import numpy as np
import pytest

import deflate_ref as dr
import pbs_plus_b200 as pg
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref
from pbs_plus_b200._lib import EINVAL
from test_deflate_cpu import cases

pytestmark = pytest.mark.gpu
SEG = dr.SEGMENT


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def ref():
    cs = cases()
    return list(cs), [cs[k] for k in cs], [dr.deflate(cs[k]) for k in cs]


def pack(parts, shift):
    offs, pos = [], shift
    for p in parts:
        offs.append(pos)
        pos += len(p) + 3                                    # ragged: every source misaligned differently
    buf = np.full(pos + 64, 0xEE, np.uint8)
    for p, o in zip(parts, offs):
        buf[o:o + len(p)] = np.frombuffer(p, np.uint8)
    return buf, np.array(offs, np.uint64), np.array([len(p) for p in parts], np.uint64)


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("out", ["host", "device"])
def test_byte_identical_to_the_restatement(eng, torch, ref, where, out):
    names, parts, want = ref
    buf, off, ln = pack(parts, 5 if where == "device" else 0)
    base = torch.from_numpy(buf).cuda() if where == "device" else buf
    got, crc = eng.deflate_batch(base, off, ln, out=out)
    for k, name in enumerate(names):
        g = got[k] if out == "host" else got[k].cpu().numpy().tobytes()
        assert g == want[k], name
        assert crc[k] == zlib.crc32(parts[k]), name


def test_pieces_through_more(eng, torch):
    data = lzref.text_corpus(5 * SEG + 999, 21).tobytes()
    whole = dr.deflate(data)
    dev = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).cuda()
    cuts = [0, SEG, 3 * SEG, len(data)]
    off = np.array(cuts[:-1], np.uint64)
    ln = np.diff(np.array(cuts, np.uint64))
    got, crc = eng.deflate_batch(dev, off, ln, more=[1, 1, 0])
    assert b"".join(got) == whole and zlib.decompress(whole, -15) == data
    c = int(crc[0])
    for k in (1, 2):
        c = pg.engine.crc32_combine(c, int(crc[k]), int(ln[k]))
    assert c == zlib.crc32(data)
    with pytest.raises(pg.PbsGpuError) as e:
        eng.deflate_batch(dev, [0], [SEG + 1], more=[1])
    assert e.value.code == EINVAL
    got, _ = eng.deflate_batch(dev, [0, 0], [0, 0], more=[1, 0])
    assert got == [b"", b"\x03\x00"]


def test_bound_on_random_data(eng, torch):
    rng = np.random.default_rng(31)
    parts = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (1, 77, 65535, SEG, 3 * SEG + 5, 9 << 20)]
    buf, off, ln = pack(parts, 0)
    got, crc = eng.deflate_batch(torch.from_numpy(buf).cuda(), off, ln)
    for p, g, c in zip(parts, got, crc):
        assert len(g) <= pg.engine.deflate_bound(len(p)) and zlib.decompress(g, -15) == p and c == zlib.crc32(p)


def half_zero_random(n, seed):
    a = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    m = n // 4096 * 4096
    a[:m].reshape(-1, 4096)[::2] = 0
    return a


@pytest.mark.parametrize("corpus", ["half_zero_random", "text", "binary"])
def test_256_mib_inflates_through_zlib(eng, torch, corpus):
    n = 256 << 20
    a = {"half_zero_random": lambda: half_zero_random(n, 1), "text": lambda: lzref.text_corpus(n, 2),
         "binary": lambda: hufref.binary_corpus(n, 3)}[corpus]()
    dev = torch.from_numpy(a).cuda()
    k = 3                                                   # three ranges, ragged ends
    cut = [0, n // 3 + 1, 2 * n // 3 + 7, n]
    off = np.array(cut[:-1], np.uint64)
    got, crc = eng.deflate_batch(dev, off, np.diff(np.array(cut, np.uint64)), out="device")
    for i in range(k):
        s = got[i].cpu().numpy().tobytes()
        piece = a[cut[i]:cut[i + 1]].tobytes()
        assert zlib.decompress(s, -15) == piece and crc[i] == zlib.crc32(piece)
        assert len(s) < len(piece)


def test_a_call_across_a_pass_edge(eng, torch):
    segs = 4096 + 37                                         # one pass is 4096 segments
    a = half_zero_random(segs * SEG - 11, 9)
    dev = torch.from_numpy(a).cuda()
    n = len(a)
    cut = [0, 5, 4096 * SEG - 3, n]                          # a range that straddles the pass edge
    got, crc = eng.deflate_batch(dev, np.array(cut[:-1], np.uint64), np.diff(np.array(cut, np.uint64)))
    for i in range(3):
        piece = a[cut[i]:cut[i + 1]].tobytes()
        assert zlib.decompress(got[i], -15) == piece and crc[i] == zlib.crc32(piece)
    # the segments near the edge match the restatement byte for byte
    lo = 4095 * SEG - 3 - 5
    tail = a[5 + lo:5 + lo + 2 * SEG].tobytes()
    g2, _ = eng.deflate_batch(dev, [5 + lo], [2 * SEG])
    assert g2[0] == dr.deflate(tail)
