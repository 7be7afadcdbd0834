"""Disk images through fixed indexes (.fidx), in one process:

  1. digest rate of an 8 GiB device-resident image (the synthetic corpus of bench.py's cfg2 recipe, 8 files of 1 GiB
     laid end to end, one stream): fixed cuts at 4 MiB and 64 KiB (pbsgpu_batch_opts.fixed_size, K3 over the chunks
     of the fixed-cut launches) next to the chunker at 4 MiB average chunks (K1 + sort + K2 + K3) on the same bytes.
     Host clock around the blocking call (it ends in a device synchronise); the calls alternate, 1 warm-up and
     `REPS` timed calls each; median GB/s.
  2. 4 KiB random reads through a reader over a .fidx of the first GiB of the image (4 MiB chunks, _z blobs):
     all chunks cached first, then reads of 1 and of 32 random 4 KiB ranges per call into pinned host memory (median
     and p99 per call); and cold reads: one 4 KiB range whose 4 MiB chunk is not cached, its blob given (median ms).

    python tools/image_bench.py [GiB, default 8] [--json PATH]

Prints the card and its power limit, and one JSON line, which --json also writes to PATH."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pbs_plus_b200 as pg  # noqa: E402

REPS = 5
ap = argparse.ArgumentParser()
ap.add_argument("gib", nargs="?", type=int, default=8)
ap.add_argument("--json", type=Path, default=None)
args = ap.parse_args()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(card)
e = pg.Engine(0)
gib = args.gib
n = gib << 30
img = torch.empty(n, dtype=torch.uint8, device="cuda")
e.corpus_fill(pg.corpus(seed=2, file_len=1 << 30, block_len=1 << 16, run_blocks=4, dup_permille=300), 0, gib, img, 1 << 30)
torch.cuda.synchronize()
res = {"card": card, "image_bytes": n}

# -- 1. digest rate ---------------------------------------------------------------------------------------------------
cfg = pg.make_config(4 << 20)
arms = {"fixed_4MiB": lambda: e.chunk_digest_batch(None, img, [0], [n], fixed_size=4 << 20),
        "fixed_64KiB": lambda: e.chunk_digest_batch(None, img, [0], [n], fixed_size=64 << 10),
        "chunker_avg_4MiB": lambda: e.chunk_digest_batch(cfg, img, [0], [n])}
times = {k: [] for k in arms}
chunks = {}
for rep in range(REPS + 1):
    for k, f in arms.items():
        t0 = time.perf_counter()
        rec = f()
        dt = time.perf_counter() - t0
        if rep:
            times[k].append(dt)
        chunks[k] = len(rec)
for k in arms:
    med = float(np.median(times[k]))
    res[k] = {"chunks": chunks[k], "median_s": med, "GB_per_s": n / med / 1e9, "min_s": min(times[k]), "max_s": max(times[k])}
    print(f"{k:18s} {chunks[k]:8d} chunks  median {med * 1e3:8.1f} ms  {n / med / 1e9:7.1f} GB/s")

# -- 2. 4 KiB random reads through an image reader ----------------------------------------------------------------------
cs = 4 << 20
m = 1 << 30
part = img[:m]
rec = e.chunk_digest_batch(None, part, [0], [m], fixed_size=cs)
off = np.arange(0, m, cs, dtype=np.uint64)
ln = np.full(len(off), cs, np.uint64)
blobs, _ = e.blob_encode_batch_z(part, off, ln)
fidx = e.fidx_build(rec["digest"], m, cs)
bbuf = np.frombuffer(b"".join(blobs), np.uint8)
bl = np.array([len(b) for b in blobs], np.uint64)
bo = np.concatenate([[0], np.cumsum(bl)[:-1]]).astype(np.uint64)
bc = np.arange(len(blobs), dtype=np.uint64)
out = e.host_alloc(32 * 4096)
rng = np.random.default_rng(3)


def read(r, offs, blob_idx):
    o = np.ascontiguousarray(offs, np.uint64)
    l = np.full(len(o), 4096, np.uint64)
    oo = np.arange(len(o), dtype=np.uint64) * np.uint64(4096)
    st = np.zeros(len(o), np.int32)
    k = len(blob_idx)
    bi = np.ascontiguousarray(blob_idx, np.uint64)
    bos, bls = bo[bi] if k else bo[:0], bl[bi] if k else bl[:0]
    e._ck(e._L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, len(o), 0, bbuf.ctypes.data, bos.ctypes.data,
                                  bls.ctypes.data, bi.ctypes.data, k, out.ctypes.data, oo.ctypes.data, st.ctypes.data, None))
    assert (st == 0).all()


with e.reader_fidx(fidx, cache_bytes=m + (64 << 20)) as r:
    read(r, [0], bc)                                                   # every chunk verified into the cache
    for per in (1, 32):
        lat = []
        for it in range(2000 // per + 50):
            t0 = time.perf_counter()
            read(r, rng.integers(0, m // 4096, per) * 4096, [])
            if it >= 50:
                lat.append(time.perf_counter() - t0)
        lat = np.array(lat)
        key = f"cached_4KiB_x{per}"
        res[key] = {"median_us": float(np.median(lat) * 1e6), "p99_us": float(np.percentile(lat, 99) * 1e6),
                    "reads_per_s": per / float(np.median(lat))}
        print(f"{key:18s} median {np.median(lat) * 1e6:8.1f} us  p99 {np.percentile(lat, 99) * 1e6:8.1f} us  "
              f"{per / np.median(lat):9.0f} reads/s")
with e.reader_fidx(fidx, cache_bytes=cs) as r:
    lat = []
    for it in range(40):
        c = int(rng.integers(0, len(blobs)))
        t0 = time.perf_counter()
        read(r, [c * cs + int(rng.integers(0, cs // 4096)) * 4096], [c])
        if it >= 5:
            lat.append(time.perf_counter() - t0)
    res["cold_4KiB"] = {"median_ms": float(np.median(lat) * 1e3), "max_ms": float(np.max(lat) * 1e3)}
    print(f"cold_4KiB          median {np.median(lat) * 1e3:8.2f} ms  max {np.max(lat) * 1e3:8.2f} ms")
e.host_free(out)
line = json.dumps(res)
print(line)
if args.json is not None:
    args.json.write_text(line + "\n")
e.close()
