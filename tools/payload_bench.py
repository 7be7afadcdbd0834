#!/usr/bin/env python
"""PayloadStreamWriter throughput (one pxar payload stream through pbsgpu_stream_*, default 2 GiB windows) with the
window products off and on: DataBlobs of the new chunks encoded at collect time (upload_blob, "z", "lze" and "lzh") and the
per-file XXH3-64 (hash_files).  The input is 64 files of 128 MiB of the device corpus (seed 4) copied to pageable host
memory, read through a reader object as a caller's io.Reader would be.  Prints one line per leg and the card it ran on.

    python tools/payload_bench.py [--files 64] [--repeat 2]
"""
import argparse
import io
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

import pbs_plus_b200 as pg  # noqa: E402
from pbs_plus_b200 import transfer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--files", type=int, default=64)
ap.add_argument("--file-mib", type=int, default=128)
ap.add_argument("--repeat", type=int, default=2)
args = ap.parse_args()

eng = pg.Engine(0)
info = eng.device_info()
try:
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0]
except Exception:
    card = f"{info['name']}, power limit not readable"
print(f"device: {card}", flush=True)

flen = args.file_mib << 20
dev = torch.empty(args.files * flen, dtype=torch.uint8, device="cuda")
eng.corpus_fill(pg.corpus(seed=4, file_len=flen), 0, args.files, dev, flen)
host = dev.cpu().numpy()
del dev
torch.cuda.empty_cache()
total = args.files * flen
cfg = pg.buzhash.NewConfig(4096)


def leg(name, **kw):
    out = {"blobs": 0, "blob_bytes": 0}

    def up(d, b):
        out["blobs"] += 1
        out["blob_bytes"] += len(b)

    best = None
    for _ in range(args.repeat):
        out["blobs"] = out["blob_bytes"] = 0
        t0 = time.perf_counter()
        w = transfer.PayloadStreamWriter(eng, cfg, eng.digest_set(1 << 20), upload_blob=up if "blob_compression" in kw else None, **kw)
        for i in range(args.files):
            f = host[i * flen:(i + 1) * flen]
            w.WriteEntryReader(transfer.Entry(f"f{i}", flen), io.BytesIO(f.data), flen)
        idx = w.Finish()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    new = sum(1 for x in idx if not x[2])
    extra = ""
    if "blob_compression" in kw:
        extra = f", {out['blobs']} blobs for {new} new chunks, blob bytes / input {out['blob_bytes'] / total:.3f}"
    if kw.get("hash_files"):
        extra += f", {len(w.backed_hashes)} file hashes"
    print(f"writer {name:12s} {total >> 30} GiB: {total / best / 2**30:6.2f} GiB/s (best of {args.repeat}, {best:.2f} s){extra}",
          flush=True)


leg("plain")
leg("blobs z", blob_compression="z")
leg("blobs lze", blob_compression="lze")
leg("blobs lzh", blob_compression="lzh")
leg("hashes", hash_files=True)
leg("z + hashes", blob_compression="z", hash_files=True)
