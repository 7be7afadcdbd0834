"""File restore into a directory: the sparse restore (PayloadReader.RestoreFiles: plan without zero chunks,
read_file_sparse, a pwrite per data extent, ftruncate) against the same files restored through ReadFileContents and
dense writes (plan, read with PAYLOAD headers, one write per file), both into a new directory, 1 GiB batches, the
reader's default 256 MiB cache.

Archives: `gib` GiB (default 8) of 64 MiB files written by PayloadStreamWriter at a 4 MiB average with _lzh blobs, in
two mixes:
  thin -- every fourth file all zeros (64 MiB, longer than the 16 MiB longest chunk); the others hold zero runs of
          4-24 MiB at unaligned offsets between 1-3 MiB of random bytes, about 90 % zeros over all;
  full -- random bytes, no zeros.
Random bytes are drawn from a pool of 1 MiB blocks placed at unaligned offsets, so the blob store stays small in host
memory; the reader still fetches and decodes every chunk index it needs.  Each restored file is checked against its
source once, outside the timed runs.

Per arm and mix: GB/s of file bytes (host clock around the blocking restore; median of `--reps`, arms alternated),
blobs fetched (= decoded), bytes copied device to host, bytes allocated on disk (st_blocks), and per run the host time
in the reader's plan calls, in the blob fetches, in its read calls, and the rest (file writes and bookkeeping).
--mix restricts the run to one archive.

    python tools/file_restore_bench.py [--gib 8] [--reps 3] [--mix thin|full|both] [--json PATH]

Prints the card and its power limit, and one JSON line, which --json also writes to PATH."""
import argparse
import io
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import pbs_plus_b200 as pg  # noqa: E402
from pbs_plus_b200 import engine, transfer  # noqa: E402

AVG = 4 << 20
FILE = 64 << 20
SLICE = 1 << 30
BLK = 1 << 20

ap = argparse.ArgumentParser()
ap.add_argument("--gib", type=int, default=8)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--mix", choices=["thin", "full", "both"], default="both")
ap.add_argument("--json", type=Path, default=None)
args = ap.parse_args()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(card, flush=True)
eng = pg.Engine(0)
n_files = (args.gib << 30) // FILE
pool = np.random.default_rng(7).integers(0, 256, (256 + 1) * BLK, dtype=np.uint8)


def file_bytes(mix: str, i: int) -> bytes:
    """File i of a mix, generated from its seed."""
    r = np.random.default_rng((1 if mix == "thin" else 2) * 1_000_003 + i)
    a = np.zeros(FILE, np.uint8)
    if mix == "thin" and i % 4 == 0:
        return a.tobytes()
    at = 0
    while at < FILE:
        n = int(r.integers(1 * BLK, 3 * BLK)) if mix == "thin" else FILE
        n = min(n, FILE - at)
        k = 0
        while k < n:   # random bytes: pool slices at unaligned offsets
            m = min(n - k, BLK)
            s = int(r.integers(0, 256 * BLK))
            a[at + k:at + k + m] = pool[s:s + m]
            k += m
        at += n
        if mix == "thin":
            at += int(r.integers(4 * BLK, 24 * BLK)) + int(r.integers(0, 4096))
    return a.tobytes()


ARCHIVES = {}
for mix in (("thin", "full") if args.mix == "both" else (args.mix,)):
    t0 = time.perf_counter()
    store = {}
    w = transfer.PayloadStreamWriter(eng, pg.make_config(AVG), upload_blob=lambda d, b, s=store: s.setdefault(d, b),
                                     blob_compression="lzh")
    entries, zero_bytes = [], 0
    for i in range(n_files):
        f = file_bytes(mix, i)
        zero_bytes += f.count(0)
        off = w.WriteEntryReader(transfer.Entry(f"f{i}", len(f)), io.BytesIO(f), len(f))
        entries.append(transfer.FileEntry(f"d{i % 8}/f{i}", 0o100644, 1_600_000_000 + i, off, len(f)))
    w.Finish()
    dirs = [transfer.DirEntry(f"d{k}", 0o40755, 1_600_000_000) for k in range(8)]
    ARCHIVES[mix] = (w.didx(), store, dirs + entries, zero_bytes)
    print(mix, "archive written:", len(w.index), "chunks,", len(store), "distinct blobs,",
          round(time.perf_counter() - t0, 1), "s", flush=True)

# the reader calls of both arms, counted and timed (host clock around each blocking call): plan, read, and the
# blob fetches; what is left of a restore's time is the host's file writes and bookkeeping
stats = {}


def timed(name: str, fn, count_d2h=None):
    def call(self, *a, **k):
        t0 = time.perf_counter()
        out = fn(self, *a, **k)
        stats[name + "_s"] += time.perf_counter() - t0
        if count_d2h:
            stats["d2h"] += count_d2h(out[1])
        return out
    return call


R = engine.Reader
R.plan, R.plan_file_sparse = timed("plan", R.plan), timed("plan", R.plan_file_sparse)
R.read = timed("read", R.read, lambda data: sum(len(d) for d in data if d is not None))
R.read_file_sparse = timed("read", R.read_file_sparse, lambda data: sum(len(p) for _, p in filter(None, data)))


def restore_sparse(pr: transfer.PayloadReader, root: Path, entries) -> None:
    pr.RestoreFiles(str(root), entries, slice_bytes=SLICE)


def restore_dense(pr: transfer.PayloadReader, root: Path, entries) -> None:
    batch, acc = [], 0
    files = [e for e in entries if isinstance(e, transfer.FileEntry)]
    for e in entries:
        if isinstance(e, transfer.DirEntry):
            os.makedirs(root / e.path, exist_ok=True)
    for k, e in enumerate(files):
        batch.append(e)
        acc += e.size
        if acc >= SLICE or k == len(files) - 1:
            for f, data in zip(batch, pr.ReadFileContents([(f.payload_offset, f.size) for f in batch])):
                with open(root / f.path, "wb") as out:
                    out.write(data)
            batch, acc = [], 0


ARMS = {"sparse": restore_sparse, "dense": restore_dense}
tmp = Path(tempfile.mkdtemp(prefix="file_restore_bench_"))


def run(arm: str, mix: str, check: bool = False) -> dict:
    didx, store, entries, _ = ARCHIVES[mix]
    root = tmp / f"{arm}-{mix}"
    stats.update(fetched=0, d2h=0, plan_s=0.0, read_s=0.0, fetch_s=0.0)

    def source(d: bytes) -> bytes:
        t0 = time.perf_counter()
        stats["fetched"] += 1
        b = store[d]
        stats["fetch_s"] += time.perf_counter() - t0
        return b

    os.sync()   # earlier runs' dirty pages are not written back inside this run's timing
    with transfer.PayloadReader(eng, didx, source) as pr:
        t0 = time.perf_counter()
        ARMS[arm](pr, root, entries)
        dt = time.perf_counter() - t0
    files = [e for e in entries if isinstance(e, transfer.FileEntry)]
    alloc = sum(os.stat(root / e.path).st_blocks * 512 for e in files)
    if check:
        for i, e in enumerate(files):
            assert (root / e.path).read_bytes() == file_bytes(mix, i), (arm, mix, e.path)
    shutil.rmtree(root)
    phases = {k: round(stats[k], 3) for k in ("plan_s", "fetch_s", "read_s")}
    phases["rest_s"] = round(dt - sum(stats[k] for k in ("plan_s", "fetch_s", "read_s")), 3)
    return {"s": dt, "fetched": stats["fetched"], "d2h": stats["d2h"], "allocated": alloc, "phases": phases}


res = {"card": card, "gib": args.gib, "file": FILE, "avg_chunk": AVG, "slice": SLICE}
try:
    for mix in ARCHIVES:
        for arm in ARMS:   # warm-up, and the one check of the restored bytes
            run(arm, mix, check=True)
    for mix in ARCHIVES:
        times = {a: [] for a in ARMS}
        for k in range(args.reps):
            for arm in (ARMS if k % 2 == 0 else reversed(ARMS)):   # ABBA order
                r = run(arm, mix)
                times[arm].append(r["s"])
                for f in ("fetched", "d2h", "allocated"):
                    res[f"{mix}_{arm}_{f}"] = r[f]
                res.setdefault(f"{mix}_{arm}_phases", []).append(r["phases"])
        for arm in ARMS:
            res[f"{mix}_{arm}_GBps"] = round(n_files * FILE / statistics.median(times[arm]) / 1e9, 3)
            res[f"{mix}_{arm}_s"] = [round(t, 3) for t in times[arm]]
        res[f"{mix}_zero_bytes"] = ARCHIVES[mix][3]
        print(mix, {k: v for k, v in res.items() if k.startswith(mix)}, flush=True)
finally:
    shutil.rmtree(tmp, ignore_errors=True)
    eng.close()
print(json.dumps(res))
if args.json:
    args.json.parent.mkdir(parents=True, exist_ok=True)
    args.json.write_text(json.dumps(res, indent=1))
