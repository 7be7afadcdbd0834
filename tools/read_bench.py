"""The archive reader (pbsgpu_reader_*) on a payload archive of the text-like and half-zero images of
tools/decode_bench.py, written as _lzh DataBlobs at 4 MiB average chunks with files of seeded sizes from 4 KiB to 8 MiB
(a PAYLOAD header before every file, a chunk boundary suggested at every file start).  All arms run in one process:

  1. restore: every file read once, 1 GiB of files per call (plan, then read with the planned blobs from pinned host
     memory), into pinned host memory through the C ABI, and through transfer.PayloadReader.ReadFileContents (Python,
     `bytes` in and out); next to pbsgpu_blob_decode_batch of the same blobs into pinned host memory (the same decode
     work without the reader's gather).  GB/s of file bytes (decoded bytes for the batch decode).
  2. cache hits: sequential 128 KiB reads over a fully cached 256 MiB region, 1 and 32 ranges per call (plan + read,
     into pinned host memory): median and p99 latency per call, GB/s.
  3. single miss: one 128 KiB read whose 4 MiB chunk is not cached, its blob given, per image: milliseconds.
  4. K14: torch.profiler kernel time of k_read_gather for 4 KiB, 128 KiB and 4 MiB pieces over 192 MiB of cached
     chunks into device memory, against a device-to-device copy of the same bytes in the same run.

    python tools/read_bench.py [GiB, default 8]"""
import ctypes as C
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import pbs_plus_b200 as pg  # noqa: E402
import zstd_lz_ref as lzref  # noqa: E402
from pbs_plus_b200 import transfer  # noqa: E402

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
e = pg.Engine(0)
L = e._L
n = int(sys.argv[1]) << 30 if len(sys.argv) > 1 else 8 << 30
half = n // 2

# -- the archive: text-like, then half-zero random; files of log-uniform sizes in [4 KiB, 8 MiB] -------------------
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
tile = torch.from_numpy(lzref.text_corpus(32 << 20, 1)).cuda()
arc = torch.empty(size, dtype=torch.uint8, device="cuda")
arc[:half] = tile.repeat(half // len(tile) + 1)[:half]
del tile
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
crc = np.zeros(nc, np.uint32)
assert L.pbsgpu_blob_encode_batch_lzh(e._h, arc.data_ptr(), starts.ctypes.data, clen.ctypes.data, nc, blobs_h.ctypes.data,
                                      boff.ctypes.data, blen.ctypes.data, crc.ctypes.data) == 0
print(f"archive: {size / 2**30:.2f} GiB, {len(sizes)} files, {nc} chunks (avg {size / nc / 2**20:.2f} MiB), "
      f"_lzh blobs {blen.sum() / size:.3f} of the input")
flen = np.array(sizes, np.uint64)
out_h = e.host_alloc(size + 16)   # the restore's files, or the batch decode's chunks


def calls():
    """the files in calls of about 1 GiB of file bytes"""
    i = 0
    while i < len(sizes):
        j, acc = i, 0
        while j < len(sizes) and (acc == 0 or acc + sizes[j] <= 1 << 30):
            acc += sizes[j]
            j += 1
        yield i, j
        i = j


out_off_all = np.concatenate([[0], np.cumsum(flen)[:-1]]).astype(np.uint64)


def restore_c(cache_bytes, max_calls=None):
    r = e.reader(didx, cache_bytes=cache_bytes)
    t0, done = time.perf_counter(), 0
    for i, j in list(calls())[:max_calls]:
        done += int(flen[i:j].sum())
        o, l, oo = files_off[i:j], flen[i:j], out_off_all[i:j]
        need = np.zeros(nc, np.uint64)
        k = C.c_uint64()
        assert L.pbsgpu_reader_plan(r._h, o.ctypes.data, l.ctypes.data, j - i, 1, need.ctypes.data, None, nc, C.byref(k)) == 0
        need = need[:k.value].copy()
        st = np.zeros(j - i, np.int32)
        bo, bl = boff[need.astype(np.int64)].copy(), blen[need.astype(np.int64)].copy()
        assert L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, j - i, 1, blobs_h.ctypes.data, bo.ctypes.data,
                                    bl.ctypes.data, need.ctypes.data, len(need), out_h.ctypes.data, oo.ctypes.data,
                                    st.ctypes.data, None) == 0
        assert (st == 0).all(), st
    dt = time.perf_counter() - t0
    r.close()
    return done, dt


def restore_py():
    mv = memoryview(np.asarray(blobs_h))
    by_digest = {bytes(rec["digest"][c]): (int(boff[c]), int(blen[c])) for c in range(nc)}
    src = lambda d: mv[by_digest[d][0]: sum(by_digest[d])]
    t0 = time.perf_counter()
    with transfer.PayloadReader(e, didx, src, cache_bytes=CACHE) as r:
        for i, j in calls():
            got = r.ReadFileContents(list(zip(files_off[i:j].tolist(), sizes[i:j])))
            assert len(got) == j - i
    return time.perf_counter() - t0


def decode_batch():
    st = np.zeros(nc, np.int32)
    dig = np.ascontiguousarray(rec["digest"])
    t0 = time.perf_counter()
    assert L.pbsgpu_blob_decode_batch(e._h, blobs_h.ctypes.data, boff.ctypes.data, blen.ctypes.data, nc, clen.ctypes.data,
                                      dig.ctypes.data, out_h.ctypes.data, starts.ctypes.data, st.ctypes.data, None) == 0
    dt = time.perf_counter() - t0
    assert (st == 0).all()
    return dt


fbytes = int(flen.sum())
CACHE = 2 << 30   # a cache that holds one call's chunks: each call decodes its blobs in one group
print(f"-- 1. restore (cache {CACHE >> 20} MiB unless stated)")
_, t = restore_c(CACHE)
# the output against the archive, on the first 64 files
got = torch.from_numpy(np.asarray(out_h)[:fbytes]).cuda()
sel = torch.cat([torch.arange(int(o) + 16, int(o) + 16 + s, device="cuda") for o, s in
                 zip(files_off[:64], sizes[:64])])
assert torch.equal(got[:sel.numel()], arc[sel]), "restore output differs from the archive"
print(f"reader, C ABI into pinned host:        {fbytes / t / 1e9:6.2f} GB/s of file bytes ({t:.2f} s)")
t = restore_py()
print(f"PayloadReader.ReadFileContents:        {fbytes / t / 1e9:6.2f} GB/s of file bytes ({t:.2f} s)")
b, t = restore_c(0, 1)
print(f"reader, default 256 MiB cache, first call: {b / t / 1e9:6.2f} GB/s of file bytes ({t:.2f} s for {b / 2**30:.2f} GiB)")
t = min(decode_batch() for _ in range(2))
print(f"blob_decode_batch into pinned host:    {size / t / 1e9:6.2f} GB/s of decoded bytes ({t:.2f} s)")

# -- 2. cache hits -------------------------------------------------------------------------------------------------
print("-- 2. cache hits (128 KiB reads over a cached region)")
r = e.reader(didx)
region_chunks = int(np.searchsorted(np.cumsum((clen + np.uint64(255)) // np.uint64(256) * np.uint64(256)), 256 << 20,
                                        side="right"))
region = int(ends[region_chunks - 1])
cs = np.arange(region_chunks, dtype=np.uint64)
st = np.zeros(32, np.int32)
assert L.pbsgpu_reader_read(r._h, None, None, 0, 0, blobs_h.ctypes.data, boff[:region_chunks].ctypes.data,
                            blen[:region_chunks].ctypes.data, cs.ctypes.data, region_chunks, None, None, None, None) == 0
region = min(region, 256 << 20)
R = 128 << 10
hit_out = e.host_alloc(32 * R)
need = np.zeros(64, np.uint64)
k = C.c_uint64()
for per in (1, 32):
    offs = np.arange(0, region - per * R + 1, per * R, dtype=np.uint64)
    lat = []
    for base_off in offs:
        o = base_off + np.arange(per, dtype=np.uint64) * np.uint64(R)
        l = np.full(per, R, np.uint64)
        oo = np.arange(per, dtype=np.uint64) * np.uint64(R)
        t0 = time.perf_counter()
        assert L.pbsgpu_reader_plan(r._h, o.ctypes.data, l.ctypes.data, per, 0, need.ctypes.data, None, 64, C.byref(k)) == 0
        assert k.value == 0
        assert L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, per, 0, None, None, None, None, 0, hit_out.ctypes.data,
                                    oo.ctypes.data, st.ctypes.data, None) == 0
        lat.append(time.perf_counter() - t0)
    lat = np.array(lat[5:])
    print(f"{per:2d} range(s) per call: median {np.median(lat) * 1e6:7.1f} us, p99 {np.percentile(lat, 99) * 1e6:7.1f} us, "
          f"{per * R * len(lat) / lat.sum() / 1e9:6.2f} GB/s ({len(lat)} calls)")
r.close()

# -- 3. single miss ------------------------------------------------------------------------------------------------
print("-- 3. single miss (one 128 KiB read, its chunk's blob given)")
for label, at in (("text-like", size // 4), ("half-zero: random half", half + (size - half) * 7 // 8),
                  ("half-zero: zero half", half + (size - half) // 4)):
    for rep in range(2):
        r = e.reader(didx)
        c = int(np.searchsorted(ends, at + rep * (16 << 20), side="right"))
        while clen[c] < 1 << 20:   # a chunk the read stays inside
            c += 1
        o = np.array([int(starts[c]) + 4096], np.uint64)
        l = np.array([R], np.uint64)
        oo = np.zeros(1, np.uint64)
        cc = np.array([c], np.uint64)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        assert L.pbsgpu_reader_read(r._h, o.ctypes.data, l.ctypes.data, 1, 0, blobs_h.ctypes.data, boff[c:c + 1].ctypes.data,
                                    blen[c:c + 1].ctypes.data, cc.ctypes.data, 1, hit_out.ctypes.data, oo.ctypes.data,
                                    st.ctypes.data, None) == 0
        dt = time.perf_counter() - t0
        assert st[0] == 0
        print(f"{label:24s} chunk {c} ({clen[c] / 2**20:.2f} MiB, blob {blen[c] / clen[c]:.3f}): {dt * 1e3:8.2f} ms")
        r.close()

# -- 4. K14 against a device-to-device copy ------------------------------------------------------------------------
print("-- 4. K14 k_read_gather against cudaMemcpy D2D (torch.profiler kernel time)")
r = e.reader(didx)
assert L.pbsgpu_reader_read(r._h, None, None, 0, 0, blobs_h.ctypes.data, boff[:region_chunks].ctypes.data,
                            blen[:region_chunks].ctypes.data, cs.ctypes.data, region_chunks, None, None, None, None) == 0
span = 192 << 20
dst = torch.empty(span, dtype=torch.uint8, device="cuda")
src = torch.empty(span, dtype=torch.uint8, device="cuda")
from torch.autograd import DeviceType  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402
for piece in (4 << 10, 128 << 10, 4 << 20):
    o = np.arange(0, span, piece, dtype=np.uint64)
    l = np.full(len(o), piece, np.uint64)
    stp = np.zeros(len(o), np.int32)
    args = (r._h, o.ctypes.data, l.ctypes.data, len(o), 0, None, None, None, None, 0, dst.data_ptr(), o.ctypes.data,
            stp.ctypes.data, None)
    assert L.pbsgpu_reader_read(*args) == 0 and (stp == 0).all()
    dst.copy_(src)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            assert L.pbsgpu_reader_read(*args) == 0
            dst.copy_(src)
        torch.cuda.synchronize()
    k14 = mc = 0.0
    nk = nm = 0
    for ev in prof.events():
        if ev.device_type != DeviceType.CUDA:
            continue
        dt = ev.time_range.elapsed_us()
        if "k_read_gather" in ev.name:
            k14 += dt
            nk += 1
        elif "Memcpy" in ev.name and "DtoD" in ev.name:
            mc += dt
            nm += 1
    if nk and nm:
        print(f"{piece >> 10:5d} KiB pieces ({len(o)} per launch): K14 {k14 / nk:8.1f} us = {span / (k14 / nk) / 1e3:6.1f} GB/s, "
              f"D2D copy {mc / nm:8.1f} us = {span / (mc / nm) / 1e3:6.1f} GB/s (copy bytes, read + write = 2x)")
    else:
        print(f"{piece >> 10} KiB pieces: events not found ({nk} K14, {nm} memcpy)",
              sorted({ev.name for ev in prof.events()})[:20])
r.close()
