"""ctypes binding of libpbsgpu.so (C ABI: include/pbsgpu.h).

The product path is the CUDA library.  There is deliberately NO fallback: if the
shared library is missing or no CUDA device is usable, loading / Engine() raises.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libpbsgpu.so"


class PbsGpuError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"pbsgpu error {code}: {msg}")
        self.code = code


EINVAL, ENOMEM, ERANGE, ECUDA, ENODEV, ESTATE = -22, -12, -34, -5, -19, -77
BATCH_EARLY_INPUT = 1  # pbsgpu_batch_opts.flags


class Cfg(C.Structure):
    _fields_ = [("avg", C.c_uint32), ("min", C.c_uint32), ("max", C.c_uint32), ("mask", C.c_uint32),
                ("break_min", C.c_uint32), ("window", C.c_uint32), ("table", C.c_uint32 * 256)]


class Chunk(C.Structure):
    _fields_ = [("stream", C.c_uint32), ("flags", C.c_uint32), ("end_off", C.c_uint64), ("digest", C.c_uint8 * 32)]


CHUNK_DTYPE = np.dtype([("stream", "<u4"), ("flags", "<u4"), ("end_off", "<u8"), ("digest", "u1", (32,))])
assert CHUNK_DTYPE.itemsize == C.sizeof(Chunk) == 48
CHUNK_KNOWN = 1
# pbsgpu_stream_blob_mode: the DataBlob encoder of a stream's new chunks (None = no blobs)
BLOB_MODES = {None: 0, "raw": 1, "z": 2, "lz": 3, "lze": 4, "lzh": 5, "lzl": 7, "lzc": 10}   # 6, 8, 9 are not assigned
# pbsgpu_blob_decode_batch: per-blob status (PBSGPU_DEC_*)
DEC_OK, DEC_BAD_MAGIC, DEC_BAD_CRC, DEC_ENCRYPTED, DEC_BAD_FRAME, DEC_BAD_SIZE, DEC_BAD_CHECKSUM, DEC_BAD_DIGEST = range(8)
DEC_BAD_TAG = 8   # pbsgpu_blob_decode_batch_enc only: the AES-256-GCM tag did not verify
# pbsgpu_reader_read: a range's chunk was neither cached nor given; a file's 16-byte PAYLOAD header did not match
DEC_MISSING, DEC_BAD_HEADER = 9, 10
READ_PAYLOAD = 1   # pbsgpu_reader_plan / _read flags: ranges are (payload offset, file size)
READ_DEFLATE_LZC = 2   # pbsgpu_reader_read_deflate only: the streams are pbsgpu_deflate_batch_lzc's
READ_SPARSE = 4   # pbsgpu_reader_plan of a .fidx reader only: zero chunks are left out
SPARSE_BLOCK = 4096   # pbsgpu_reader_read_sparse: holes are image-aligned blocks of this size, or their parts in a range


class DevInfo(C.Structure):
    _fields_ = [("device", C.c_int32), ("sm_count", C.c_int32), ("cc_major", C.c_int32), ("cc_minor", C.c_int32),
                ("total_mem", C.c_uint64), ("free_mem", C.c_uint64), ("name", C.c_char * 64)]


class Timing(C.Structure):
    _fields_ = [("scan_ms", C.c_float), ("sort_ms", C.c_float), ("resolve_ms", C.c_float), ("sha_ms", C.c_float),
                ("set_ms", C.c_float), ("total_ms", C.c_float), ("scan_t0", C.c_float), ("scan_t1", C.c_float),
                ("sha_t0", C.c_float), ("sha_t1", C.c_float), ("sha_long_ms", C.c_float), ("sha_bulk_ms", C.c_float),
                ("bytes", C.c_uint64), ("chunks", C.c_uint64),
                ("candidates", C.c_uint64), ("scan_launches", C.c_uint32), ("sha_launches", C.c_uint32),
                ("other_launches", C.c_uint32), ("reruns", C.c_uint32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class BatchOpts(C.Structure):
    """pbsgpu_batch_opts: digest set, suggested boundaries, per-stream XXH3 output, encrypt mode's keyed digests."""
    _fields_ = [("size", C.c_uint32), ("flags", C.c_uint32), ("set", C.c_void_p), ("forced_stream", C.c_void_p),
                ("forced_off", C.c_void_p), ("n_forced", C.c_uint64), ("stream_xxh3", C.c_void_p), ("crypt", C.c_void_p)]


class BatchOptsFixed(BatchOpts):
    """pbsgpu_batch_opts in its current layout: BatchOpts (the layout up to `crypt`, which the library still accepts)
    plus `fixed_size`, the fixed cuts of a .fidx image (0 = the chunker)."""
    _fields_ = [("fixed_size", C.c_uint32)]


FIDX_MAGIC = bytes([0x2f, 0x7f, 0x41, 0xed, 0x91, 0xfd, 0x0f, 0xcd])   # sha256("Proxmox Backup fixed sized chunk index v1.0")[:8]


class Corpus(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("file_len", C.c_uint64), ("block_len", C.c_uint64),
                ("run_blocks", C.c_uint32), ("dup_permille", C.c_uint32), ("edit_mode", C.c_uint32),
                ("edit_thresh16", C.c_uint32), ("edit_seed", C.c_uint64)]


class ZipEntry(C.Structure):
    """pbsgpu_zip_entry: one entry of the zip container (name bytes, Unix st_mode, mtime, method, CRC, sizes, the
    offset of its local header)."""
    _fields_ = [("name", C.c_void_p), ("name_len", C.c_uint32), ("mode", C.c_uint32), ("mtime", C.c_int64),
                ("method", C.c_uint32), ("crc", C.c_uint32), ("comp_size", C.c_uint64), ("size", C.c_uint64),
                ("offset", C.c_uint64)]


DEFLATE_SEGMENT = 128 * 1024   # pbsgpu_deflate_batch: a piece that a later call continues is a multiple of this


# Every symbol include/pbsgpu.h declares (tests assert the .so exports all of them) and its ctypes signature: the
# argument types, or (argument types, result type) where the result is not int.
_vp, _u32p, _u64p = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
_SIGNATURES = {
    "pbsgpu_version": [],
    "pbsgpu_open": [C.c_int, C.POINTER(_vp)],
    "pbsgpu_close": ([_vp], None),
    "pbsgpu_strerror": ([_vp], C.c_char_p),
    "pbsgpu_device_info": [_vp, C.POINTER(DevInfo)],
    "pbsgpu_set_profiling": [_vp, C.c_int],
    "pbsgpu_partition_info": [_vp, C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "pbsgpu_scan_partition_sms": [_vp],
    "pbsgpu_set_kernel_variant": [_vp, C.c_int],
    "pbsgpu_config": [C.c_uint32, _u32p, C.POINTER(Cfg)],
    "pbsgpu_config_kib": [C.c_uint32, _u32p, C.POINTER(Cfg)],
    "pbsgpu_default_table": ([], _u32p),
    "pbsgpu_chunk_digest_batch": [_vp, C.POINTER(Cfg), _vp, _vp, _vp, C.c_uint32, _vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_batch_submit": [_vp, C.POINTER(Cfg), _vp, _vp, _vp, C.c_uint32, C.POINTER(_vp)],
    "pbsgpu_batch_wait": [_vp, _vp, C.c_uint64, _u64p, C.POINTER(Timing)],
    "pbsgpu_chunk_digest_batch_ex": [_vp, C.POINTER(Cfg), _vp, _vp, _vp, C.c_uint32, C.POINTER(BatchOpts), _vp, C.c_uint64, _u64p],
    "pbsgpu_batch_submit_ex": [_vp, C.POINTER(Cfg), _vp, _vp, _vp, C.c_uint32, C.POINTER(BatchOpts), C.POINTER(_vp)],
    "pbsgpu_batch_free": ([_vp], None),
    "pbsgpu_batch_wait_input": [_vp],
    "pbsgpu_batch_input_done": [_vp],
    "pbsgpu_scan_batch": [_vp, C.POINTER(Cfg), _vp, _vp, _vp, C.c_uint32, _vp, C.c_uint64, _vp, _u64p],
    "pbsgpu_sha256_batch": [_vp, _vp, _vp, _vp, C.c_uint32, _vp],
    "pbsgpu_sha256_keyed_batch": [_vp, _vp, _vp, _vp, _vp, C.c_uint32, _vp],
    "pbsgpu_stream_crypt": [_vp, _vp, _vp],
    "pbsgpu_stream_open": [_vp, C.POINTER(Cfg), _vp, C.POINTER(_vp)],
    "pbsgpu_stream_write": [_vp, _vp, C.c_uint64],
    "pbsgpu_stream_poll": [_vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_stream_finish": [_vp],
    "pbsgpu_stream_close": ([_vp], None),
    "pbsgpu_stream_reserve": [_vp, C.POINTER(_vp)],
    "pbsgpu_stream_commit": [_vp, C.c_uint64],
    "pbsgpu_stream_slot_bytes": ([_vp], C.c_uint64),
    "pbsgpu_stream_suggest": [_vp, C.c_uint64],
    "pbsgpu_stream_position": ([_vp], C.c_uint64),
    "pbsgpu_stream_blob_mode": [_vp, C.c_int],
    "pbsgpu_stream_poll_blobs": [_vp, _vp, C.c_uint64, _vp, C.c_uint64, _u64p],
    "pbsgpu_stream_hash_range": [_vp, C.c_uint64, C.c_uint64],
    "pbsgpu_stream_poll_hashes": [_vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_set_create": [_vp, C.c_uint64, C.POINTER(_vp)],
    "pbsgpu_set_destroy": ([_vp], None),
    "pbsgpu_set_insert": [_vp, _vp, C.c_uint64, _vp],
    "pbsgpu_set_probe": [_vp, _vp, C.c_uint64, _vp],
    "pbsgpu_set_count": [_vp, _u64p],
    "pbsgpu_set_seed_didx": [_vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_set_allgather": [_vp, _vp, _vp, C.c_uint64, _vp],
    "pbsgpu_nccl_unique_id": [_vp],
    "pbsgpu_nccl_comm_create": [_vp, _vp, C.c_int, C.c_int, C.POINTER(_vp)],
    "pbsgpu_nccl_comm_destroy": ([_vp], None),
    "pbsgpu_didx_size": ([C.c_uint64], C.c_uint64),
    "pbsgpu_didx_build": [_vp, _vp, C.c_uint64, _vp, C.c_int64, _vp, C.c_uint64],
    "pbsgpu_didx_parse": [_vp, _vp, C.c_uint64, _vp, _vp, C.c_uint64, _u64p, C.c_int],
    "pbsgpu_fidx_size": ([C.c_uint64], C.c_uint64),
    "pbsgpu_fidx_build": [_vp, _vp, C.c_uint64, C.c_uint64, C.c_uint64, _vp, C.c_int64, _vp, C.c_uint64],
    "pbsgpu_fidx_parse": [_vp, _vp, C.c_uint64, _u64p, _u64p, _vp, C.c_uint64, _u64p, C.c_int],
    "pbsgpu_set_seed_fidx": [_vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_reader_open_fidx": [_vp, _vp, C.c_uint64, _vp, C.c_uint64, C.POINTER(_vp)],
    "pbsgpu_crc32_batch": [_vp, _vp, _vp, _vp, C.c_uint32, _vp],
    "pbsgpu_blob_header": ([C.c_uint32, _vp], None),
    "pbsgpu_blob_size": ([C.c_uint64], C.c_uint64),
    "pbsgpu_blob_encode_batch": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp],
    "pbsgpu_blob_encode_batch_z": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_encode_batch_lz": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_encode_batch_lze": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_encode_batch_lzh": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_encode_batch_lzl": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_encode_batch_lzc": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_crypt_create": [_vp, _vp, C.POINTER(_vp)],
    "pbsgpu_crypt_destroy": ([_vp], None),
    "pbsgpu_blob_size_enc": ([C.c_uint64], C.c_uint64),
    "pbsgpu_blob_encode_batch_enc": [_vp, _vp, C.c_int, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_decode_batch": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp],
    "pbsgpu_blob_decode_batch_enc": [_vp, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp],
    "pbsgpu_reader_open": [_vp, _vp, C.c_uint64, _vp, C.c_uint64, C.POINTER(_vp)],
    "pbsgpu_reader_close": ([_vp], None),
    "pbsgpu_reader_size": ([_vp], C.c_uint64),
    "pbsgpu_reader_plan": [_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_reader_read": [_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp],
    "pbsgpu_deflate_bound": ([C.c_uint64], C.c_uint64),
    "pbsgpu_deflate_batch": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp],
    "pbsgpu_deflate_batch_lzc": [_vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp],
    "pbsgpu_crc32_combine": ([C.c_uint32, C.c_uint32, C.c_uint64], C.c_uint32),
    "pbsgpu_reader_read_deflate": [_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp,
                                   _vp, _vp],
    "pbsgpu_reader_read_sparse": [_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp,
                                  C.c_uint64, _vp, _vp, _vp],
    "pbsgpu_reader_plan_file_sparse": [_vp, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, C.c_uint64, _u64p],
    "pbsgpu_reader_read_file_sparse": [_vp, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp, C.c_uint32, _vp, _vp,
                                       _vp, C.c_uint64, _vp, _vp, _vp],
    "pbsgpu_zip_local_header": ([C.POINTER(ZipEntry), _vp, C.c_uint64], C.c_uint64),
    "pbsgpu_zip_data_descriptor": ([C.POINTER(ZipEntry), _vp, C.c_uint64], C.c_uint64),
    "pbsgpu_zip_directory": ([_vp, C.c_uint64, C.c_uint64, _vp, C.c_uint64], C.c_uint64),
    "pbsgpu_xxh3_batch": [_vp, _vp, _vp, _vp, C.c_uint32, _vp],
    "pbsgpu_chunk_digest_batch_xxh3": [_vp, C.POINTER(Cfg), _vp, _vp, _vp, C.c_uint32, _vp, _vp, C.c_uint64, _u64p, _vp],
    "pbsgpu_host_alloc": ([_vp, C.c_uint64], _vp),
    "pbsgpu_host_free": ([_vp, _vp], None),
    "pbsgpu_corpus_fill": [_vp, C.POINTER(Corpus), C.c_uint64, C.c_uint32, _vp, C.c_uint64],
}
SYMBOLS = list(_SIGNATURES)

_lib = None


def lib() -> C.CDLL:
    """Load libpbsgpu.so (fails loudly when the CUDA extension has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} not found: the CUDA extension is the product and there is no fallback. "
            "Build it with `python -m pbs_plus_b200.build` (or __graft_entry__.build()).")
    L = C.CDLL(str(LIB_PATH))
    for name, sig in _SIGNATURES.items():
        fn = getattr(L, name)
        fn.argtypes, fn.restype = sig if isinstance(sig, tuple) else (sig, C.c_int)
    _lib = L
    return L
