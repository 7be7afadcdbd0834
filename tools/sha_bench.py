#!/usr/bin/env python
"""K3 alone at saturation: SHA-256 of N equal ranges (no length imbalance, no tail).
usage: python tools/sha_bench.py [range_kib] [total_gib]"""
import sys, time
from pathlib import Path
import numpy as np
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch
import pbs_plus_b200 as pg

rk = int(sys.argv[1]) if len(sys.argv) > 1 else 256
tg = int(sys.argv[2]) if len(sys.argv) > 2 else 32
eng = pg.Engine(0)
n = (tg << 30) // (rk << 10)
buf = torch.empty(tg << 30, dtype=torch.uint8, device="cuda")
eng.corpus_fill(pg.corpus(seed=9, file_len=tg << 30), 0, 1, buf, tg << 30)
off = np.arange(n, dtype=np.uint64) * (rk << 10) + (3 if len(sys.argv) > 3 else 0)   # optional misalignment
ln = np.full(n, (rk << 10) - 64, dtype=np.uint64)
eng.sha256_batch(buf, off, ln)
torch.cuda.synchronize()
best = 1e9
for _ in range(3):
    t0 = time.perf_counter(); d = eng.sha256_batch(buf, off, ln); dt = time.perf_counter() - t0
    best = min(best, dt)
import hashlib
chk = hashlib.sha256(buf[int(off[5]): int(off[5]) + int(ln[5])].cpu().numpy().tobytes()).digest() == bytes(d[5])
print(f"ranges {n} x {rk} KiB: {ln.sum()/best/1e9:.1f} GB/s  ({best*1e3:.1f} ms) ok={chk}")
