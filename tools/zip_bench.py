"""The zip restore's Deflate stage and the zip restore itself, all arms in one process:

  1. pbsgpu_deflate_batch and pbsgpu_deflate_batch_lzc on 8 GiB device-resident images (64 ranges of 128 MiB, device
     out): the half-zero random, tests/zstd_lz_ref.text_corpus and tests/zstd_huf_ref.binary_corpus generators (a
     32 MiB tile repeated; segments are coded independently, so the repeat gives no cross-tile matches).  GB/s of
     input and output / input.
  2. host zlib (raw Deflate) levels 1, 4 and 6 on one core, 8 samples of 8 MiB of each image, for context only.
  3. a zip restore of an 8 GiB _lzh payload archive (text-like, then half-zero, files of 4 KiB to 8 MiB, as
     tools/read_bench.py builds it) through transfer.ZipWriter, default and lzc=True, into a byte-counting sink,
     against PayloadReader.ReadFileContents of the same files in the same run.  GB/s of file bytes.

Prints the card and its power limit, then one JSON line.

    python tools/zip_bench.py [GiB, default 8]"""
import io
import json
import stat
import subprocess
import sys
import time
import zlib
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import pbs_plus_b200 as pg  # noqa: E402
import zstd_huf_ref as hufref  # noqa: E402
import zstd_lz_ref as lzref  # noqa: E402
from pbs_plus_b200 import engine as E, transfer  # noqa: E402

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(card)
e = pg.Engine(0)
n = int(sys.argv[1]) << 30 if len(sys.argv) > 1 else 8 << 30
TILE = 32 << 20
result = {"card": card, "bytes": n}


def image(kind: str) -> torch.Tensor:
    if kind == "half_zero_random":
        a = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
        a.view(-1, 4096)[::2] = 0
        return a
    t = lzref.text_corpus(TILE, 1) if kind == "text" else hufref.binary_corpus(TILE, 2)
    return torch.from_numpy(t).cuda().repeat(n // TILE)


# -- 1 + 2 ---------------------------------------------------------------------------------------------------------
RANGE = 128 << 20
off = np.arange(0, n, RANGE, dtype=np.uint64)
ln = np.full(len(off), RANGE, np.uint64)
bound = np.array([E.deflate_bound(RANGE)] * len(off), np.uint64)
ooff = np.concatenate([[0], np.cumsum(bound)[:-1]]).astype(np.uint64)
for kind in ("half_zero_random", "text", "binary"):
    a = image(kind)
    out = torch.empty(int(bound.sum()), dtype=torch.uint8, device="cuda")
    olen = np.zeros(len(off), np.uint64)
    crc = np.zeros(len(off), np.uint32)
    gpu = {}
    for arm in ("deflate_batch", "deflate_batch_lzc"):
        best = None
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e._ck(getattr(e._L, "pbsgpu_" + arm)(e._h, a.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off), None,
                                                 out.data_ptr(), ooff.ctypes.data, olen.ctypes.data, crc.ctypes.data))
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        s0 = out[:int(olen[0])].cpu().numpy().tobytes()
        assert zlib.decompress(s0, -15) == a[:RANGE].cpu().numpy().tobytes(), (kind, arm)
        gpu[arm] = (n / best / 1e9, float(olen.sum()) / n)
    h = a[:64 << 20].cpu().numpy()
    host = {}
    for lvl in (1, 4, 6):
        t0 = time.perf_counter()
        outb = 0
        for k in range(8):
            c = zlib.compressobj(lvl, zlib.DEFLATED, -15)
            outb += len(c.compress(h[k << 23:(k + 1) << 23].tobytes()) + c.flush())
        dt = time.perf_counter() - t0
        host[f"zlib{lvl}"] = {"GBps": (64 << 20) / dt / 1e9, "ratio": outb / (64 << 20)}
    result[kind] = {"deflate_batch_GBps": gpu["deflate_batch"][0], "ratio": gpu["deflate_batch"][1],
                    "deflate_batch_lzc_GBps": gpu["deflate_batch_lzc"][0], "ratio_lzc": gpu["deflate_batch_lzc"][1],
                    "host_one_core": host}
    print(f"{kind:16s} " + ", ".join(f"{arm} {g:7.2f} GB/s, out/in {r:.4f}" for arm, (g, r) in gpu.items()) + "; host "
          + ", ".join(f"zlib-{lvl} {host[f'zlib{lvl}']['GBps']:.3f} GB/s ({host[f'zlib{lvl}']['ratio']:.4f})"
                      for lvl in (1, 4, 6)))
    del a, out
    torch.cuda.empty_cache()

# -- 3. zip restore of a payload archive -----------------------------------------------------------------------------
rng = np.random.default_rng(11)
sizes, pos = [], 16
while True:
    s = int(np.exp(rng.uniform(np.log(4096), np.log(8 << 20))))
    if pos + 16 + s + 16 > n:
        break
    sizes.append(s)
    pos += 16 + s
files_off = np.zeros(len(sizes), np.uint64)
p = 16
for i, s in enumerate(sizes):
    files_off[i] = p
    p += 16 + s
size = p + 16
half = size // 2
arc = torch.empty(size, dtype=torch.uint8, device="cuda")
tile = torch.from_numpy(lzref.text_corpus(TILE, 1)).cuda()
arc[:half] = tile.repeat(half // TILE + 1)[:half]
arc[half:] = torch.randint(0, 256, (size - half,), dtype=torch.uint8, device="cuda")
arc[half: half + (size - half) // 2] = 0
hdr = np.zeros((len(sizes), 16), np.uint8)
hdr[:, :8] = np.frombuffer(transfer.PXAR_PAYLOAD.to_bytes(8, "little"), np.uint8)
hdr[:, 8:] = (np.array(sizes, np.uint64) + np.uint64(16)).view(np.uint8).reshape(-1, 8)
idx = torch.from_numpy(files_off.astype(np.int64)).cuda()[:, None] + torch.arange(16, device="cuda")[None, :]
arc[idx.reshape(-1)] = torch.from_numpy(hdr.reshape(-1)).cuda()
torch.cuda.synchronize()
rec = e.chunk_digest_batch(pg.make_config(4 << 20), arc, [0], [size],
                           forced=(np.zeros(len(sizes) - 1, np.uint32), files_off[1:]))
ends = rec["end_off"].astype(np.uint64)
starts = np.concatenate([[0], ends[:-1]]).astype(np.uint64)
clen = ends - starts
nc = len(ends)
didx = e.didx_build(rec)
boff = np.concatenate([[0], np.cumsum(clen + np.uint64(12))[:-1]]).astype(np.uint64)
blobs_h = e.host_alloc(int((clen + np.uint64(12)).sum()))
blen = np.zeros(nc, np.uint64)
bcrc = np.zeros(nc, np.uint32)
assert e._L.pbsgpu_blob_encode_batch_lzh(e._h, arc.data_ptr(), starts.ctypes.data, clen.ctypes.data, nc,
                                         blobs_h.ctypes.data, boff.ctypes.data, blen.ctypes.data, bcrc.ctypes.data) == 0
del arc, tile
torch.cuda.empty_cache()
mv = memoryview(np.asarray(blobs_h))
by_digest = {bytes(rec["digest"][c]): (int(boff[c]), int(blen[c])) for c in range(nc)}
src = lambda d: mv[by_digest[d][0]: sum(by_digest[d])]
fbytes = sum(sizes)
files = [(f"f{i}", stat.S_IFREG | 0o644, 1_700_000_000, int(o), s) for i, (o, s) in enumerate(zip(files_off, sizes))]
CACHE = 2 << 30


class Count(io.RawIOBase):
    def __init__(self):
        self.n = 0

    def writable(self):
        return True

    def write(self, b):
        self.n += len(b)
        return len(b)


def zip_restore(lzc=False):
    sink = Count()
    t0 = time.perf_counter()
    with transfer.PayloadReader(e, didx, src, cache_bytes=CACHE) as r:
        z = transfer.ZipWriter(r, sink, lzc=lzc)
        z.AddFiles(files)
        z.Close()
    return time.perf_counter() - t0, sink.n


def read_files():
    t0 = time.perf_counter()
    with transfer.PayloadReader(e, didx, src, cache_bytes=CACHE) as r:
        i = 0
        while i < len(files):
            j, acc = i, 0
            while j < len(files) and (acc == 0 or acc + sizes[j] <= 1 << 30):
                acc += sizes[j]
                j += 1
            assert len(r.ReadFileContents([(f[3], f[4]) for f in files[i:j]])) == j - i
            i = j
    return time.perf_counter() - t0


tz, zbytes = min(zip_restore() for _ in range(2))
tc, cbytes = min(zip_restore(True) for _ in range(2))
tr = min(read_files() for _ in range(2))
result["zip_restore"] = {"files": len(files), "file_bytes": fbytes, "zip_bytes": zbytes, "zip_GBps": fbytes / tz / 1e9,
                         "zip_bytes_lzc": cbytes, "zip_lzc_GBps": fbytes / tc / 1e9, "read_files_GBps": fbytes / tr / 1e9}
print(f"zip restore: {len(files)} files, {fbytes / 2**30:.2f} GiB -> zip {zbytes / fbytes:.4f} of the file bytes: "
      f"ZipWriter {fbytes / tz / 1e9:.2f} GB/s; lzc=True {cbytes / fbytes:.4f} at {fbytes / tc / 1e9:.2f} GB/s; "
      f"ReadFileContents {fbytes / tr / 1e9:.2f} GB/s")
print(json.dumps(result))
