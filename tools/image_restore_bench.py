"""Disk-image restore: the sparse restore (transfer.restore_image: plan without zero chunks, read_sparse, a pwrite per
data extent) against the same image restored through plain reads (plan, read, one pwrite per slice -- what ReadAt
slices do), both into a new file, 1 GiB slices, the reader's default 256 MiB cache.

Images: `gib` GiB (default 8) of 4 MiB chunks with _lzh blobs, in two mixes:
  thin -- 75 % zero chunks, 10 % half-zero chunks (random first half), the rest random;
  full -- random chunks, no zeros.
The data chunks are drawn from a pool of distinct chunks, so the blob store stays small in host memory; the reader
still fetches and decodes every chunk index it needs, as for distinct chunks.  Each restored file is checked against
the image once, outside the timed runs.

Per arm and mix: GB/s of image bytes (host clock around the blocking restore; median of `--reps`, arms alternated),
blobs fetched (= decoded; also how many of them were the zero chunk's), and bytes copied device to host.
`--profile` instead runs one restore of each mix per arm under torch.profiler and reports the summed CUDA time of K17
(k_zero_map), K14 (k_read_gather) and all kernels.

    python tools/image_restore_bench.py [--gib 8] [--reps 3] [--profile] [--json PATH]

Prints the card and its power limit, and one JSON line, which --json also writes to PATH."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pbs_plus_b200 as pg  # noqa: E402
from pbs_plus_b200 import _lib, engine, transfer  # noqa: E402

CS = 4 << 20
SLICE = 1 << 30
POOL_DATA, POOL_HALF = 64, 32

ap = argparse.ArgumentParser()
ap.add_argument("--gib", type=int, default=8)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--profile", action="store_true")
ap.add_argument("--json", type=Path, default=None)
args = ap.parse_args()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(card, flush=True)
eng = pg.Engine(0)
n_chunks = (args.gib << 30) // CS

# the chunk pool: random chunks, half-zero chunks, and the zero chunk; one _lzh blob per distinct chunk
rng = np.random.default_rng(7)
pool = rng.integers(0, 256, (POOL_DATA + POOL_HALF + 1, CS), dtype=np.uint8)
pool[POOL_DATA:POOL_DATA + POOL_HALF, CS // 2:] = 0
pool[-1] = 0
ZERO, flat = len(pool) - 1, pool.reshape(-1)
off = np.arange(len(pool), dtype=np.uint64) * CS
ln = np.full(len(pool), CS, np.uint64)
pool_dig = [bytes(d) for d in eng.sha256_batch(flat, off, ln)]
assert pool_dig[ZERO] == hashlib.sha256(bytes(CS)).digest()
store = dict(zip(pool_dig, eng.blob_encode_batch_lzh(flat, off, ln)[0]))


def layout(mix: str) -> np.ndarray:
    """Pool index per chunk of the image."""
    r = np.random.default_rng(11 if mix == "thin" else 12)
    if mix == "full":
        return r.integers(0, POOL_DATA, n_chunks)
    u = r.random(n_chunks)
    return np.where(u < 0.75, ZERO, np.where(u < 0.85, POOL_DATA + r.integers(0, POOL_HALF, n_chunks),
                                             r.integers(0, POOL_DATA, n_chunks)))


IMAGES = {}
for mix in ("thin", "full"):
    lay = layout(mix)
    fidx = eng.fidx_build(b"".join(pool_dig[p] for p in lay), n_chunks * CS, CS)
    data_bytes = int(sum(CS if p < POOL_DATA else CS // 2 if p < ZERO else 0 for p in lay))
    IMAGES[mix] = (lay, fidx, data_bytes)

stats = {}
_read_sparse, _read = engine.Reader.read_sparse, engine.Reader.read


def counted_read_sparse(self, *a, **k):
    st, data, bst = _read_sparse(self, *a, **k)
    stats["d2h"] += sum(len(p) for _, p in filter(None, data))
    return st, data, bst


def counted_read(self, *a, **k):
    st, data, bst = _read(self, *a, **k)
    stats["d2h"] += sum(len(d) for d in data if d is not None)
    return st, data, bst


engine.Reader.read_sparse, engine.Reader.read = counted_read_sparse, counted_read


def source(d: bytes) -> bytes:
    stats["fetched"] += 1
    stats["zero_fetched"] += d == pool_dig[ZERO]
    return store[d]


def restore_sparse(fidx: bytes, fd: int) -> None:
    transfer.restore_image(eng, fidx, source, fd, slice_bytes=SLICE)


def restore_read(fidx: bytes, fd: int) -> None:
    with eng.reader_fidx(fidx) as r:
        size = r.size
        for at in range(0, size, SLICE):
            n = min(SLICE, size - at)
            chunks, dig = r.plan([at], [n])
            st, data, _ = r.read([at], [n], {int(c): source(bytes(d)) for c, d in zip(chunks, dig)})
            assert st[0] == _lib.DEC_OK
            view, done = memoryview(data[0]), 0
            while done < n:
                done += os.pwrite(fd, view[done:], at + done)


ARMS = {"sparse": restore_sparse, "read": restore_read}
tmp = Path(tempfile.mkdtemp(prefix="restore_bench_"))


def run(arm: str, mix: str, check: bool = False) -> dict:
    lay, fidx, _ = IMAGES[mix]
    path = tmp / f"{arm}-{mix}.img"
    stats.update(fetched=0, zero_fetched=0, d2h=0)
    os.sync()   # earlier runs' dirty pages are not written back inside this run's timing
    fd = os.open(path, os.O_RDWR | os.O_CREAT | os.O_TRUNC, 0o600)
    try:
        t0 = time.perf_counter()
        ARMS[arm](fidx, fd)
        dt = time.perf_counter() - t0
        if check:
            for c, p in enumerate(lay):
                assert os.pread(fd, CS, c * CS) == pool[p].tobytes(), (arm, mix, c)
    finally:
        os.close(fd)
        path.unlink()
    return {"s": dt, "fetched": stats["fetched"], "zero_fetched": stats["zero_fetched"], "d2h": stats["d2h"]}


res = {"card": card, "gib": args.gib, "chunk": CS, "slice": SLICE}
try:
    for mix in IMAGES:
        for arm in ARMS:   # warm-up, and the one check of the restored bytes
            run(arm, mix, check=True)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for mix in IMAGES:
            for arm in ARMS:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run(arm, mix)
                ev = [e for e in prof.key_averages() if e.device_type.name == "CUDA"]
                tot = lambda f: sum(e.device_time_total for e in ev if f(e.key)) / 1e3   # noqa: E731 (ms)
                res[f"{mix}_{arm}_profile_ms"] = {"k17_zero_map": tot(lambda k: "k_zero_map" in k),
                                                  "k14_read_gather": tot(lambda k: "k_read_gather" in k),
                                                  "all_kernels": tot(lambda k: not k.startswith("Memcpy") and
                                                                     not k.startswith("Memset"))}
                print(mix, arm, res[f"{mix}_{arm}_profile_ms"], flush=True)
    else:
        for mix in IMAGES:
            times = {a: [] for a in ARMS}
            for k in range(args.reps):
                for arm in (ARMS if k % 2 == 0 else reversed(ARMS)):   # ABBA order
                    r = run(arm, mix)
                    times[arm].append(r["s"])
                    for f in ("fetched", "zero_fetched", "d2h"):
                        res[f"{mix}_{arm}_{f}"] = r[f]
            for arm in ARMS:
                res[f"{mix}_{arm}_GBps"] = round(n_chunks * CS / statistics.median(times[arm]) / 1e9, 3)
                res[f"{mix}_{arm}_s"] = [round(t, 3) for t in times[arm]]
            res[f"{mix}_data_bytes"] = IMAGES[mix][2]
            print(mix, {k: v for k, v in res.items() if k.startswith(mix)}, flush=True)
finally:
    tmp.rmdir()
    eng.close()
print(json.dumps(res))
if args.json:
    args.json.parent.mkdir(parents=True, exist_ok=True)
    args.json.write_text(json.dumps(res, indent=1))
