"""f3 read side microbench: pbsgpu_blob_decode_batch over the DataBlobs of 4 MiB chunks of the four 8 GiB images of
tools/blob_bench.py (half-zero random, text-like, binary-like, repeated).  Per image, the blobs of three encoders --
_lzh and _lzl (this engine) and libzstd level 1 (pyarrow, compressed on the host before any timing) -- lie in device
memory, and the call runs twice: verify only (out = NULL, expected digests given) and with the chunks copied into
pinned host memory.  A fourth arm, "lzh-enc", decodes encrypted _lzh blobs (pbsgpu_blob_encode_batch_enc) with
pbsgpu_blob_decode_batch_enc and keyed digests the same two ways.  Rates are GB/s of decoded bytes, the best of 3 runs.
For context only: libzstd's single-thread decode rate on the HOST CPU over a 64 MiB sample of the level-1 blobs.

    python tools/decode_bench.py [GiB per image, default 8]"""
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pyarrow as pa
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import pbs_plus_b200 as pg  # noqa: E402
import zstd_huf_ref as hufref  # noqa: E402
import zstd_ldm_ref as ldmref  # noqa: E402
import zstd_lz_ref as lzref  # noqa: E402
from oracle import pyref  # noqa: E402

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
e = pg.Engine(0)
L_ = e._L
n = int(sys.argv[1]) << 30 if len(sys.argv) > 1 else 8 << 30
CH = 4 << 20
nc = n // CH
off = np.arange(0, n, CH, dtype=np.uint64)
ln = np.full(nc, CH, dtype=np.uint64)
boff = np.arange(nc, dtype=np.uint64) * np.uint64(CH + 44)
blobs_h = e.host_alloc(nc * (CH + 44))
blen = np.zeros(nc, dtype=np.uint64)
crc = np.zeros(nc, dtype=np.uint32)
dec_h = e.host_alloc(n)
status = np.zeros(nc, dtype=np.int32)
dig_out = np.zeros((nc, 32), dtype=np.uint8)
KEY = os.urandom(32)
iv = np.frombuffer(os.urandom(16 * nc), dtype=np.uint8)


def images():
    d = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
    d[n // 8: n // 8 * 5] = 0
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


def libzstd_blobs(d):
    """level-1 DataBlobs of every chunk, packed at boff / blen in blobs_h (the smaller of frame and raw chunk)"""
    host = d.cpu().numpy()
    codec = pa.Codec("zstd", compression_level=1)

    def one(i):
        chunk = host[i * CH:(i + 1) * CH]
        fr = codec.compress(chunk, asbytes=True)
        if len(fr) < CH:
            b = pyref.BLOB_MAGIC_COMPRESSED + zlib.crc32(fr).to_bytes(4, "little") + fr
        else:
            b = pyref.BLOB_MAGIC_UNCOMPRESSED + zlib.crc32(chunk).to_bytes(4, "little") + chunk.tobytes()
        blobs_h[int(boff[i]):int(boff[i]) + len(b)] = np.frombuffer(b, np.uint8)
        blen[i] = len(b)
    with ThreadPoolExecutor(16) as ex:
        list(ex.map(one, range(nc)))
    sample = [codec.compress(host[i * CH:(i + 1) * CH], asbytes=True) for i in range(0, nc, max(1, nc // 16))]
    t0 = time.perf_counter()
    for fr in sample:
        pa.decompress(fr, decompressed_size=CH, codec="zstd")
    return len(sample) * CH / (time.perf_counter() - t0) / 1e9


for label, d in images():
    torch.cuda.synchronize()
    want = e.sha256_batch(d, off, ln)
    print(f"-- {label} image, {n / 2**30:.0f} GiB")
    for enc in ("lzh", "lzh-enc", "lzl", "libzstd-1"):
        host_rate = None
        if enc == "libzstd-1":
            host_rate = libzstd_blobs(d)
        elif enc == "lzh-enc":
            # an engine of its own: closing it returns the decryption stage, so the other arms keep their device memory
            ee = pg.Engine(0)
            cr = ee.crypt(KEY)
            want_keyed = ee.sha256_keyed_batch(cr, d, off, ln)
            rc = L_.pbsgpu_blob_encode_batch_enc(ee._h, cr._h, 5, d.data_ptr(), off.ctypes.data, ln.ctypes.data, nc,
                                                 iv.ctypes.data, blobs_h.ctypes.data, boff.ctypes.data, blen.ctypes.data,
                                                 crc.ctypes.data)
            assert rc == 0, rc
        else:
            rc = getattr(L_, "pbsgpu_blob_encode_batch_" + enc)(e._h, d.data_ptr(), off.ctypes.data, ln.ctypes.data, nc,
                                                                blobs_h.ctypes.data, boff.ctypes.data, blen.ctypes.data,
                                                                crc.ctypes.data)
            assert rc == 0, rc
        bd = torch.from_numpy(np.asarray(blobs_h)).cuda()
        res = {}
        for mode, outp in (("verify only", None), ("into pinned host", dec_h.ctypes.data)):
            best = 1e9
            for rep in range(3):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if enc == "lzh-enc":
                    rc = L_.pbsgpu_blob_decode_batch_enc(ee._h, cr._h, bd.data_ptr(), boff.ctypes.data, blen.ctypes.data, nc,
                                                         ln.ctypes.data, want_keyed.ctypes.data, outp, off.ctypes.data,
                                                         status.ctypes.data, dig_out.ctypes.data)
                else:
                    rc = L_.pbsgpu_blob_decode_batch(e._h, bd.data_ptr(), boff.ctypes.data, blen.ctypes.data, nc,
                                                     ln.ctypes.data, want.ctypes.data, outp, off.ctypes.data,
                                                     status.ctypes.data, dig_out.ctypes.data)
                best = min(best, time.perf_counter() - t0)
                assert rc == 0 and (status == 0).all(), (rc, np.unique(status))
            res[mode] = n / best / 1e9
        del bd
        if enc == "lzh-enc":
            cr.close()
            ee.close()
        torch.cuda.empty_cache()
        ctx = f"; libzstd host decode, one thread: {host_rate:.2f} GB/s" if host_rate else ""
        print(f"{enc}: blobs {blen.sum() / n:.4f} of the input; decode {res['verify only']:.2f} GB/s verify only, "
              f"{res['into pinned host']:.2f} GB/s into pinned host{ctx}", flush=True)
    del d
    torch.cuda.empty_cache()
