"""The zip container functions (pbsgpu_zip_*, host only) read back by Python's zipfile: stored and zlib-deflated data,
directories and symlinks, non-ASCII names, modes and mtimes, zip64 sizes, a local header beyond 4 GiB (a sparse
file), and more than 65535 entries; plus the declarations."""
import io
import re
import stat
import zipfile
import zlib
from pathlib import Path

import pytest

from pbs_plus_b200 import _lib, engine as E

ROOT = Path(__file__).resolve().parent.parent


class Archive:
    """An archive written the way a restore writes one: local header, content, data descriptor, and the directory."""

    def __init__(self, f):
        self.f, self.entries = f, []

    def add(self, name: str, mode: int, mtime: int, content: bytes = b"", deflate: bool = False, size=None, crc=None,
            hole: int = 0):
        comp = content
        if deflate:
            c = zlib.compressobj(6, zlib.DEFLATED, -15)
            comp = c.compress(content) + c.flush()
        e = E.zip_entry(name.encode(), mode, mtime, 8 if deflate else 0, zlib.crc32(content) if crc is None else crc,
                        len(comp) + hole, len(content) + hole if size is None else size, self.f.tell())
        self.f.write(E.zip_local_header(e))
        if hole:
            self.f.seek(hole, io.SEEK_CUR)
        self.f.write(comp)
        self.f.write(E.zip_data_descriptor(e))
        self.entries.append(e)

    def close(self):
        self.f.write(E.zip_directory(self.entries, self.f.tell()))


def test_zipfile_reads_files_dirs_symlinks_names_modes_mtimes():
    buf = io.BytesIO()
    a = Archive(buf)
    text = b"the quick brown fox " * 5000
    a.add("dir/", stat.S_IFDIR | 0o750, 1_700_000_000)
    a.add("dir/empty/", stat.S_IFDIR | 0o700, 1_600_000_001)
    a.add("dir/text.txt", stat.S_IFREG | 0o644, 1_700_000_123, text, deflate=True)
    a.add("dir/stored.bin", stat.S_IFREG | 0o600, 1_500_000_000, bytes(range(256)) * 3)
    a.add("dir/empty.txt", stat.S_IFREG | 0o644, 1_700_000_000, b"", deflate=True)
    a.add("dir/ünïcödé ☃.txt", stat.S_IFREG | 0o640, 1_700_000_000, b"snow", deflate=True)
    a.add("dir/link", stat.S_IFLNK | 0o777, 1_700_000_000, b"text.txt")
    a.add("old.txt", stat.S_IFREG | 0o644, 100, b"before 1980", deflate=True)
    a.close()
    z = zipfile.ZipFile(io.BytesIO(buf.getvalue()))
    assert z.testzip() is None
    info = {i.filename: i for i in z.infolist()}
    assert set(info) == {"dir/", "dir/empty/", "dir/text.txt", "dir/stored.bin", "dir/empty.txt", "dir/ünïcödé ☃.txt",
                         "dir/link", "old.txt"}
    assert z.read("dir/text.txt") == text and info["dir/text.txt"].compress_type == zipfile.ZIP_DEFLATED
    assert z.read("dir/stored.bin") == bytes(range(256)) * 3 and info["dir/stored.bin"].compress_type == zipfile.ZIP_STORED
    assert z.read("dir/empty.txt") == b"" and z.read("dir/ünïcödé ☃.txt") == b"snow"
    assert info["dir/ünïcödé ☃.txt"].flag_bits & 0x800 and not info["dir/text.txt"].flag_bits & 0x800
    assert info["dir/"].is_dir() and info["dir/"].external_attr == (stat.S_IFDIR | 0o750) << 16 | 0x10
    assert info["dir/text.txt"].external_attr >> 16 == stat.S_IFREG | 0o644
    assert info["dir/text.txt"].create_system == 3 and info["dir/text.txt"].flag_bits & 0x8
    assert not info["dir/"].flag_bits & 0x8
    assert stat.S_ISLNK(info["dir/link"].external_attr >> 16) and z.read("dir/link") == b"text.txt"
    assert info["dir/text.txt"].date_time == (2023, 11, 14, 22, 15, 22)   # 1_700_000_123 UTC, seconds halved
    assert info["old.txt"].date_time == (1980, 1, 1, 0, 0, 0)
    ext = info["dir/text.txt"].extra
    assert ext[:5] == b"\x55\x54\x05\x00\x01" and int.from_bytes(ext[5:9], "little") == 1_700_000_123


def test_extended_timestamp_only_in_range():
    for mtime, has in ((0, True), ((1 << 32) - 1, True), (-1, False), (1 << 32, False)):
        e = E.zip_entry(b"f", stat.S_IFREG | 0o644, mtime, 8)
        assert (b"\x55\x54" in E.zip_local_header(e)) == has, mtime
    e = E.zip_entry(b"f", stat.S_IFREG | 0o644, 1 << 40, 8)
    assert E.zip_local_header(e)[10:14] == bytes.fromhex("7dbf") + bytes.fromhex("9fff")   # 2107-12-31 23:59:58


def test_data_descriptor_sizes():
    small = E.zip_entry(b"f", 0o100644, 0, 8, 0x12345678, 10, 20)
    assert E.zip_data_descriptor(small) == bytes.fromhex("504b0708") + (0x12345678).to_bytes(4, "little") + \
        (10).to_bytes(4, "little") + (20).to_bytes(4, "little")
    for cs, us in ((10, 0xFFFFFFFF), (0xFFFFFFFF, 10)):
        assert len(E.zip_data_descriptor(E.zip_entry(b"f", 0o100644, 0, 8, 0, cs, us))) == 24
    assert E.zip_data_descriptor(E.zip_entry(b"d/", 0o40755, 0)) == b""


def test_zip64_sizes_and_a_local_header_beyond_4_gib(tmp_path):
    size = (1 << 32) + 1
    crc = E.crc32_combine(0, zlib.crc32(bytes(1 << 20)), 1 << 20)
    for _ in range(12):   # CRC-32 of 2^32 zeros by doubling, then one more zero byte
        crc = E.crc32_combine(crc, crc, 1 << (20 + _))
    crc = E.crc32_combine(crc, zlib.crc32(b"\0"), 1)
    path = tmp_path / "big.zip"
    with open(path, "wb") as f:
        a = Archive(f)
        a.add("zeros.bin", stat.S_IFREG | 0o644, 1_700_000_000, b"", hole=size, size=size, crc=crc)
        a.add("after.txt", stat.S_IFREG | 0o644, 1_700_000_000, b"past 4 GiB" * 100, deflate=True)
        a.close()
    z = zipfile.ZipFile(path)
    info = {i.filename: i for i in z.infolist()}
    assert info["zeros.bin"].file_size == size == info["zeros.bin"].compress_size and info["zeros.bin"].CRC == crc
    assert info["after.txt"].header_offset > 1 << 32
    assert z.read("after.txt") == b"past 4 GiB" * 100
    with z.open("zeros.bin") as r:
        assert r.read(1 << 16) == bytes(1 << 16)


def test_more_than_65535_entries():
    buf = io.BytesIO()
    a = Archive(buf)
    n = 70_000
    for k in range(n):
        a.add(f"f{k}", stat.S_IFREG | 0o644, 1_700_000_000, str(k).encode())
    a.close()
    z = zipfile.ZipFile(io.BytesIO(buf.getvalue()))
    names = z.namelist()
    assert len(names) == n and names[-1] == f"f{n - 1}"
    assert z.read("f65536") == b"65536" and z.read(f"f{n - 1}") == str(n - 1).encode()


def test_zip_and_deflate_are_declared_and_the_header_stays_plain_c():
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    for name in ("pbsgpu_deflate_bound", "pbsgpu_deflate_batch", "pbsgpu_crc32_combine", "pbsgpu_zip_local_header",
                 "pbsgpu_zip_data_descriptor", "pbsgpu_zip_directory"):
        assert re.search(rf"\b{name}\(", hdr) and name in _lib.SYMBOLS, name
    assert "typedef struct pbsgpu_zip_entry {" in hdr
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = '#include "pbsgpu.h"\nint main(void) { pbsgpu_zip_entry e = {0}; return (int)pbsgpu_deflate_bound(e.size); }\n'
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", str(ROOT / "include"), "-x", "c", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
