"""Encrypt-mode microbench: K11 (AES-256-GCM) over 8 GiB of resident 4 MiB chunks, encrypting and decrypting (the
blobs it wrote, read back by pbsgpu_blob_decode_batch_enc, verify only), next to K6 (CRC-32) on the same bytes, from
torch.profiler kernel times; and the wall time of the _lzh encoder against encrypted _lzh on the text-like
image (tests/zstd_lz_ref.py text_corpus, 32 MiB repeated), both into pinned host memory through the raw C calls.
Then the keyed against the plain batch path on cfg2's files.  Prints the card's name and power limit first."""
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import pbs_plus_b200 as pg  # noqa: E402
import zstd_lz_ref as lzref  # noqa: E402

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
GIB = int(os.environ.get("CRYPT_BENCH_GIB", "8"))
e = pg.Engine(0)
L_ = e._L
cr = e.crypt(os.urandom(32))
n, CH = GIB << 30, 4 << 20
off = np.arange(0, n, CH, dtype=np.uint64)
ln = np.full(len(off), CH, dtype=np.uint64)
boff = np.arange(len(off), dtype=np.uint64) * np.uint64(CH + 44)
out = e.host_alloc(int(len(off)) * (CH + 44))
blen = np.zeros(len(off), dtype=np.uint64)
crc = np.zeros(len(off), dtype=np.uint32)
iv = np.frombuffer(os.urandom(16 * len(off)), dtype=np.uint8)


def enc(d, mode):
    rc = L_.pbsgpu_blob_encode_batch_enc(e._h, cr._h, mode, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off),
                                         iv.ctypes.data, out.ctypes.data, boff.ctypes.data, blen.ctypes.data, crc.ctypes.data)
    assert rc == 0, rc


def lzh(d):
    rc = L_.pbsgpu_blob_encode_batch_lzh(e._h, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off), out.ctypes.data,
                                         boff.ctypes.data, blen.ctypes.data, crc.ctypes.data)
    assert rc == 0, rc


def dec(bd):
    rc = L_.pbsgpu_blob_decode_batch_enc(e._h, cr._h, bd.data_ptr(), boff.ctypes.data, blen.ctypes.data, len(off),
                                         ln.ctypes.data, None, None, None, status.ctypes.data, None)
    assert rc == 0 and (status == 0).all(), (rc, np.unique(status))


d = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
enc(d, 1)   # warm-up: tables, pools, module load
bd = torch.from_numpy(np.asarray(out)).cuda()   # the raw encrypted blobs, read back below
status = np.zeros(len(off), dtype=np.int32)
dec(bd)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(3):
        enc(d, 1)
    for _ in range(3):
        dec(bd)
    for _ in range(3):
        rc = L_.pbsgpu_crc32_batch(e._h, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off), crc.ctypes.data)
        assert rc == 0
    torch.cuda.synchronize()
times = {}
for ev in prof.events():
    if ev.device_type.name == "CUDA" and ("k_gcm" in ev.name or "k_crc32" in ev.name):
        times.setdefault(ev.name.split("(")[0], []).append(ev.device_time_total / 1e3)
print(f"-- random image, {GIB} GiB of 4 MiB chunks, kernel times (ms, per call)")
for k, v in sorted(times.items()):
    if "<true>" in k:   # the decrypt kernel runs once per decode pass: its time per call is the sum over the passes
        per_call = sum(v) / 3
        print(f"{k}: {per_call:.2f} ms per call ({len(v)} launches in 3 calls) -> {n / per_call / 1e6:.1f} GB/s")
        continue
    per_call = sorted(v)[len(v) // 2]
    print(f"{k}: median {per_call:.2f} ms over {len(v)} launches -> {n / per_call / 1e6:.1f} GB/s")
for rep in range(3):
    t0 = time.perf_counter()
    enc(d, 1)
    dt = time.perf_counter() - t0
print(f"blob_encode_batch_enc(raw) end to end: {n / dt / 1e9:.1f} GB/s ({dt * 1e3:.0f} ms, third run)")
del d, bd
torch.cuda.empty_cache()
tile = torch.from_numpy(lzref.text_corpus(32 << 20, 1)).cuda()
d = tile.repeat(n // len(tile))
del tile
print(f"-- text-like image, {GIB} GiB")
for name, fn in (("blob_encode_batch_lzh", lambda: lzh(d)), ("blob_encode_batch_enc(lzh)", lambda: enc(d, 5))):
    for rep in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        dt = time.perf_counter() - t0
    print(f"{name}: {n / dt / 1e9:.2f} GB/s of input ({dt * 1e3:.0f} ms, third run), output / input {blen.sum() / n:.4f}")
del d
# keyed against plain digests on cfg2's files (64 MiB each, seed 2, 4 MiB average chunks), resident, alternated
n_files, flen = 64 * GIB, 64 << 20               # 512 files = 32 GiB at the default 8
d = torch.empty(n_files * flen, dtype=torch.uint8, device="cuda")
e.corpus_fill(pg.corpus(seed=2, file_len=flen), 0, n_files, d, flen)
torch.cuda.synchronize()
foff = np.arange(n_files, dtype=np.uint64) * flen
flen_a = np.full(n_files, flen, np.uint64)
cfg = pg.make_config(4 << 20)
times = {"plain": [], "keyed": []}
e.chunk_digest_batch(cfg, d, foff, flen_a)
e.chunk_digest_batch(cfg, d, foff, flen_a, crypt=cr)
for rep in range(5):
    for name, kw in (("plain", {}), ("keyed", {"crypt": cr})):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e.chunk_digest_batch(cfg, d, foff, flen_a, **kw)
        times[name].append(time.perf_counter() - t0)
print(f"-- cfg2 files, {n_files} x 64 MiB resident, chunk_digest_batch at 4 MiB average, 5 alternated calls each")
for name, v in times.items():
    v = sorted(v)
    print(f"{name}: median {v[2] * 1e3:.1f} ms ({n_files * flen / v[2] / 2**30:.1f} GiB/s), min {v[0] * 1e3:.1f}, max {v[-1] * 1e3:.1f}")
e.host_free(out)
cr.close()
e.close()
