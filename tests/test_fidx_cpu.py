"""Fixed indexes (.fidx) without a GPU: the magic re-derived from its label, the restatement's round trips, every
rejection of pbsgpu_fidx_parse (the checksum is checked on the GPU, in test_gpu_fidx.py), and the layout of
pbsgpu_batch_opts with `fixed_size` next to the layouts before it."""
import ctypes as C
import hashlib
import subprocess
from pathlib import Path

import numpy as np
import pytest

import fidx_ref
from pbs_plus_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent
CS = 64 << 10


def c_parse(image: bytes, cap=None):
    """pbsgpu_fidx_parse without a context and without verify -> (rc, size, chunk_size, n, digests)."""
    L = _lib.lib()
    a = np.frombuffer(bytes(image), dtype=np.uint8)
    size, cs, n = C.c_uint64(), C.c_uint64(), C.c_uint64()
    cap = (len(a) // 32) if cap is None else cap
    dig = np.zeros((max(cap, 1), 32), dtype=np.uint8)
    rc = L.pbsgpu_fidx_parse(None, a.ctypes.data, len(a), C.byref(size), C.byref(cs), dig.ctypes.data, cap, C.byref(n), 0)
    return rc, size.value, cs.value, n.value, dig[: n.value]


def image_of(size: int, cs: int = CS, seed: int = 0) -> bytes:
    data = np.random.default_rng(seed).integers(0, 256, size, dtype=np.uint8).tobytes()
    return fidx_ref.fidx_build(fidx_ref.chunk_digests(data, cs), size, cs, bytes(range(16)), 1_700_000_000)


def test_magic_is_rederived_from_its_label():
    assert hashlib.sha256(fidx_ref.FIDX_LABEL).digest()[:8] == fidx_ref.FIDX_MAGIC == _lib.FIDX_MAGIC
    assert c_parse(image_of(1))[0] == 0   # the library's magic is the same bytes


@pytest.mark.parametrize("size", [0, 1, CS - 1, CS, CS + 1, 5 * CS, 5 * CS + 17])
def test_restatement_round_trips_and_the_library_reads_it(size):
    img = image_of(size, seed=size)
    assert len(img) == _lib.lib().pbsgpu_fidx_size(fidx_ref.n_chunks(size, CS)) == 4096 + 32 * -(-size // CS)
    s, cs, dig = fidx_ref.fidx_parse(img)
    assert (s, cs) == (size, CS) and fidx_ref.fidx_build(dig, s, cs, bytes(range(16)), 1_700_000_000) == img
    rc, s2, cs2, n, d2 = c_parse(img)
    assert (rc, s2, cs2, n) == (0, size, CS, len(dig)) and d2.tobytes() == b"".join(dig)


def test_parse_counts_without_a_buffer_and_reports_a_short_one():
    img = image_of(3 * CS + 5)
    L = _lib.lib()
    a = np.frombuffer(img, dtype=np.uint8)
    n = C.c_uint64()
    assert L.pbsgpu_fidx_parse(None, a.ctypes.data, len(a), None, None, None, 0, C.byref(n), 0) == 0 and n.value == 4
    assert c_parse(img, cap=3)[0] == _lib.ERANGE


def _with(img: bytes, at: int, field: bytes) -> bytes:
    b = bytearray(img)
    b[at:at + len(field)] = field
    return bytes(b)


def test_every_rejection():
    img = image_of(3 * CS + 5)
    u64 = lambda v: int(v).to_bytes(8, "little")
    bad = {
        "wrong magic": _with(img, 0, b"\x1c\x91\x4e\xa5\x19\xba\xb3\xcd"),     # the .didx magic
        "chunk_size 0": _with(img, 72, u64(0)),
        "chunk_size 2^32": _with(img, 72, u64(1 << 32)),
        "one digest short": img[:-32],
        "one digest extra": img + bytes(32),
        "a byte short": img[:-1],
        "size of one more chunk": _with(img, 64, u64(4 * CS + 1)),
        "size of one chunk less": _with(img, 64, u64(3 * CS)),
        "header only": img[:4095],
        "huge size": _with(img, 64, u64((1 << 64) - 1)),
    }
    for what, b in bad.items():
        assert c_parse(b)[0] == _lib.EINVAL, what
        with pytest.raises(ValueError):
            fidx_ref.fidx_parse(b, verify=False)
    flipped = _with(img, 4096 + 40, bytes([img[4096 + 40] ^ 1]))
    with pytest.raises(ValueError):
        fidx_ref.fidx_parse(flipped)                       # the library's verify runs on the GPU (test_gpu_fidx.py)
    assert c_parse(flipped)[0] == 0                        # without verify the table is taken as it is
    assert _with(img, 64, u64(3 * CS + 1)) != img and c_parse(_with(img, 64, u64(3 * CS + 1)))[0] == 0   # same n


def test_null_arguments_are_einval():
    L = _lib.lib()
    n = C.c_uint64()
    h = C.c_void_p()
    assert L.pbsgpu_fidx_parse(None, None, 4096, None, None, None, 0, C.byref(n), 0) == _lib.EINVAL
    assert L.pbsgpu_fidx_build(None, None, 0, 0, CS, bytes(16), 0, bytes(4096), 4096) == _lib.EINVAL
    assert L.pbsgpu_set_seed_fidx(None, bytes(4096), 4096, C.byref(n)) == _lib.EINVAL
    assert L.pbsgpu_reader_open_fidx(None, bytes(4096), 4096, None, 0, C.byref(h)) == _lib.EINVAL and not h.value


def test_batch_opts_layouts(tmp_path):
    """`fixed_size` follows `crypt`: the layout before it (size 56, BatchOpts) and the one before `crypt` (48) are what
    older callers pass; the library reads each by its size (GPU test)."""
    assert _lib.BatchOpts.crypt.offset == 48 and C.sizeof(_lib.BatchOpts) == 56
    assert _lib.BatchOptsFixed.fixed_size.offset == 56 and C.sizeof(_lib.BatchOptsFixed) == 64
    src = tmp_path / "t.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "pbsgpu.h"
int main(void) {
    printf("%zu %zu %zu\n", offsetof(pbsgpu_batch_opts, crypt), offsetof(pbsgpu_batch_opts, fixed_size), sizeof(pbsgpu_batch_opts));
    printf("%llu\n", (unsigned long long)pbsgpu_fidx_size(3));
    return 0;
}
''')
    exe = tmp_path / "t.bin"
    lib = ROOT / "pbs_plus_b200"
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-I", str(ROOT / "include"), "-o", str(exe), str(src),
                           f"-L{lib}", "-lpbsgpu", f"-Wl,-rpath,{lib}"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert out == ["48", "56", "64", str(4096 + 96)]


def test_fidx_surface_is_declared():
    hdr = " ".join((ROOT / "include" / "pbsgpu.h").read_text().split())
    for decl in ("uint64_t pbsgpu_fidx_size(uint64_t n_chunks);",
                 "int pbsgpu_fidx_build(pbsgpu_ctx *ctx, const uint8_t *digests, uint64_t n, uint64_t size, uint64_t chunk_size, "
                 "const uint8_t uuid[16], int64_t ctime, uint8_t *out, uint64_t cap);",
                 "int pbsgpu_fidx_parse(pbsgpu_ctx *ctx, const uint8_t *fidx, uint64_t bytes, uint64_t *size, uint64_t *chunk_size, "
                 "uint8_t *digests, uint64_t cap, uint64_t *n_entries, int verify);",
                 "int pbsgpu_set_seed_fidx(pbsgpu_set *set, const uint8_t *fidx, uint64_t bytes, uint64_t *n_entries);",
                 "int pbsgpu_reader_open_fidx(pbsgpu_ctx *ctx, const uint8_t *fidx, uint64_t bytes, const pbsgpu_crypt *crypt, "
                 "uint64_t cache_bytes, pbsgpu_reader **out);",
                 "uint32_t fixed_size;"):
        assert decl in hdr, decl
