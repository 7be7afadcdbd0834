"""f3 microbench: DataBlob assembly for 4 MiB chunks of an 8 GiB device-resident image into PINNED host memory through
the raw C calls (no Python-side allocation or slicing inside the timed region).  Four images: random bytes with half of
them zero runs, a text-like image (tests/zstd_lz_ref.py text_corpus, 32 MiB repeated), a binary-like one
(tests/zstd_huf_ref.py binary_corpus, 32 MiB repeated) and one with repeats far beyond one block (every 4 MiB chunk is
4 copies of 1 MiB of binary_corpus with 2000 random byte edits, tests/zstd_ldm_ref.py repeated_image).  For each: GB/s
of input and output / input of every encoder, and for context libzstd levels 1 and 3 (pyarrow, one host thread) on a
64 MiB host sample of the same image (8 MiB from each GiB), their ratios and single-thread rates on the HOST CPU.
blob_encode_batch_enc_lzc is the encrypted call in _lzc mode (random IVs).

    python tools/blob_bench.py [call ...]     # e.g. blob_encode_batch_lzh blob_encode_batch_lzc; default: every call"""
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import pbs_plus_b200 as pg  # noqa: E402
import zstd_huf_ref as hufref  # noqa: E402
import zstd_ldm_ref as ldmref  # noqa: E402
import zstd_lz_ref as lzref  # noqa: E402

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
e = pg.Engine(0)
L_ = e._L
n = 8 << 30
CH = 4 << 20
off = np.arange(0, n, CH, dtype=np.uint64)
ln = np.full(len(off), CH, dtype=np.uint64)
boff = (np.arange(len(off), dtype=np.uint64) * np.uint64(CH + 44))   # room for an encrypted blob's header
out = e.host_alloc(int(len(off)) * (CH + 44))
ivs = np.random.default_rng(0).integers(0, 256, 16 * len(off), dtype=np.uint8)
crypt = e.crypt(bytes(range(32)))
blen = np.zeros(len(off), dtype=np.uint64)
crc = np.zeros(len(off), dtype=np.uint32)


CALLS = sys.argv[1:] or ["crc32_batch", "blob_encode_batch", "blob_encode_batch_z", "blob_encode_batch_lz",
                         "blob_encode_batch_lze", "blob_encode_batch_lzh", "blob_encode_batch_lzl",
                         "blob_encode_batch_lzc", "blob_encode_batch_enc_lzc"]


def images():
    d = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
    d[1 << 30: 5 << 30] = 0
    yield "half-zero random", d
    del d
    tile = torch.from_numpy(lzref.text_corpus(32 << 20, 1)).cuda()
    yield "text-like", tile.repeat(n // len(tile))
    del tile
    tile = torch.from_numpy(hufref.binary_corpus(32 << 20, 1)).cuda()
    yield "binary-like", tile.repeat(n // len(tile))
    del tile
    tile = torch.from_numpy(ldmref.repeated_image(hufref.binary_corpus(1 << 20, 1))).cuda()
    yield "repeated", tile.repeat(n // len(tile))


for label, d in images():
    torch.cuda.synchronize()
    print(f"-- {label} image, {n / 2**30:.0f} GiB")
    for name in CALLS:
        for rep in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if name == "crc32_batch":
                rc = L_.pbsgpu_crc32_batch(e._h, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off), crc.ctypes.data)
                size = 0
            elif name == "blob_encode_batch_enc_lzc":
                rc = L_.pbsgpu_blob_encode_batch_enc(e._h, crypt._h, 10, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off),
                                                     ivs.ctypes.data, out.ctypes.data, boff.ctypes.data, blen.ctypes.data,
                                                     crc.ctypes.data)
                size = int(blen.sum())
            elif name == "blob_encode_batch":
                rc = L_.pbsgpu_blob_encode_batch(e._h, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off), out.ctypes.data,
                                                 boff.ctypes.data, crc.ctypes.data)
                size = len(off) * (CH + 12)
            else:
                rc = getattr(L_, "pbsgpu_" + name)(e._h, d.data_ptr(), off.ctypes.data, ln.ctypes.data, len(off), out.ctypes.data,
                                                   boff.ctypes.data, blen.ctypes.data, crc.ctypes.data)
                size = int(blen.sum())
            dt = time.perf_counter() - t0
            assert rc == 0, rc
        ratio = f", output / input {size / n:.4f}" if size else ""
        print(f"{name}: {n / dt / 1e9:.1f} GB/s of input ({dt * 1e3:.0f} ms, third run), {size / 2**30:.2f} GiB written to "
              f"pinned host memory{ratio}")
    try:
        import pyarrow as pa
        sample = b"".join(d[k * (n // 8): k * (n // 8) + (8 << 20)].cpu().numpy().tobytes() for k in range(8))
        for level in (1, 3):
            t0 = time.perf_counter()
            z = pa.Codec("zstd", compression_level=level).compress(sample, asbytes=True)
            dt = time.perf_counter() - t0
            print(f"libzstd level {level} (host CPU, one thread, 8 x 8 MiB sample): output / input {len(z) / len(sample):.4f}, "
                  f"{len(sample) / dt / 1e9:.2f} GB/s")
    except ImportError:
        print("libzstd: pyarrow not available")
    del d
crypt.close()
e.host_free(out)
e.close()
