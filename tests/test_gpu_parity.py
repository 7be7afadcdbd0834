"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle.

Oracle = restatement (oracle/oracle.c); boundaries are bit-exact against IT
("parity unpinned" against the absent Go module); digests additionally against hashlib.
"""
import hashlib
import json
import os
from pathlib import Path

import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, size=n, dtype=np.uint8)


def to_dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pack(arrs, align=256, lead=0):
    """Pack host arrays into one buffer; returns (buf, off, len)."""
    offs, pos = [], lead
    for a in arrs:
        offs.append(pos)
        pos += (len(a) + align - 1) // align * align if align > 1 else len(a)
    buf = np.zeros(max(pos, 1) + 64, dtype=np.uint8)
    for a, o in zip(arrs, offs):
        buf[o:o + len(a)] = a
    return buf, np.array(offs, dtype=np.uint64), np.array([len(a) for a in arrs], dtype=np.uint64)


def oracle_ends(cfg_o, arrs):
    ends, first = [], [0]
    for a in arrs:
        e = oracle.chunk_ends(cfg_o, a).tolist()
        ends += e
        first.append(len(ends))
    return ends, first


RAGGED = [0, 1, 63, 64, 65, 100, 255, 256, 257, 1023, 1024, 1025, 4095, 8703, 8704, 8705, 8704 * 2 - 1, 8704 * 2,
          8704 * 2 + 1, 8704 * 3 + 17, 50_000, 123_457]


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("avg", [256, 1024, 4096])
def test_scan_ragged_streams_match_oracle(eng, torch, variant, avg):
    eng.set_kernel_variant(variant)
    try:
        arrs = [rnd(n, 100 + i) for i, n in enumerate(RAGGED)]
        buf, off, ln = pack(arrs)
        ends, first = eng.scan_batch(pg.make_config(avg), to_dev(torch, buf), off, ln)
        ref_e, ref_f = oracle_ends(oracle.config(avg), arrs)
        assert ends.tolist() == ref_e and first.tolist() == ref_f
    finally:
        eng.set_kernel_variant(0)


@pytest.mark.parametrize("variant", [0, 1])
def test_scan_unaligned_offsets(eng, torch, variant):
    """Stream starts at every residue mod 16 (TMA needs 16 B; the kernel must cope)."""
    eng.set_kernel_variant(variant)
    try:
        arrs = [rnd(30_000 + 7 * i, 200 + i) for i in range(17)]
        buf, off, ln = pack(arrs, align=1, lead=1)
        assert len({int(o) % 16 for o in off}) > 8
        ends, first = eng.scan_batch(pg.make_config(1024), to_dev(torch, buf), off, ln)
        ref_e, ref_f = oracle_ends(oracle.config(1024), arrs)
        assert ends.tolist() == ref_e and first.tolist() == ref_f
    finally:
        eng.set_kernel_variant(0)


def test_scan_large_random_stream_all_restatements(eng, torch):
    data = rnd(32 << 20, 7)
    for avg in (4096, 65536, 1 << 20):
        ends, _ = eng.scan_batch(pg.make_config(avg), to_dev(torch, data), [0], [len(data)])
        assert ends.tolist() == oracle.chunk_ends(oracle.config(avg), data).tolist()


def test_forced_cuts_on_constant_data(eng, torch):
    data = np.zeros(1_000_000, dtype=np.uint8)
    ends, _ = eng.scan_batch(pg.make_config(1024), to_dev(torch, data), [0], [len(data)])
    assert ends.tolist() == list(range(4096, 1_000_000, 4096)) + [1_000_000]


def test_dense_candidates_overflow_rerun_is_exact(eng, torch):
    """A table that makes ~50 % of positions candidates overflows the statistically
    sized candidate buffer; the library reruns with a larger one and stays exact."""
    t = np.zeros(256, dtype=np.uint32)
    t[0] = 0xFFFFFFFF
    data = np.random.default_rng(3).integers(0, 2, size=600_000, dtype=np.uint8)
    ends, _ = eng.scan_batch(pg.make_config(512, t), to_dev(torch, data), [0], [len(data)])
    assert ends.tolist() == oracle.chunk_ends(oracle.config(512, t), data).tolist()


@pytest.mark.parametrize("entry", ["device_batch", "staged_batch", "stream"])
def test_dense_candidates_overflow_rerun_is_exact_in_every_entry_point(eng, torch, entry):
    """The same overflow through the other entry points that rerun an overflowed job: one device job over all
    streams, host input staged in several groups, and a stream cut into several windows (front half rerun only)."""
    t = np.zeros(256, dtype=np.uint32)
    t[0] = 0xFFFFFFFF
    data = np.random.default_rng(3).integers(0, 2, size=600_000, dtype=np.uint8)
    cfg, cfg_o = pg.make_config(512, t), oracle.config(512, t)
    if entry == "device_batch":
        arrs = [data[:250_000], data[250_000:]]
        buf, off, ln = pack(arrs)
        rec = eng.chunk_digest_batch(cfg, to_dev(torch, buf), off, ln)
        assert rec.tobytes() == oracle.chunk_digest_streams(cfg_o, arrs).tobytes()
    elif entry == "staged_batch":
        arrs = [data[i:i + 150_000] for i in range(0, len(data), 150_000)]
        e = _engine_with_env({"PBSGPU_STAGE_BYTES": str(1 << 18)})     # one stream per staging group
        try:
            rec = e.chunk_digest_streams(cfg, arrs)
        finally:
            e.close()
        assert rec.tobytes() == oracle.chunk_digest_streams(cfg_o, arrs).tobytes()
    else:
        e = _engine_with_env({"PBSGPU_STREAM_WINDOW": str(1 << 17)})   # five windows
        try:
            st = e.stream(cfg)
            st.write(data)
            rec = st.finish()
            st.close()
        finally:
            e.close()
        assert rec.tobytes() == oracle.chunk_digest(cfg_o, data).tobytes()


def test_custom_table(eng, torch):
    t = np.random.default_rng(9).integers(0, 2**32, size=256, dtype=np.uint32)
    data = rnd(2_000_000, 11)
    ends, _ = eng.scan_batch(pg.make_config(2048, t), to_dev(torch, data), [0], [len(data)])
    assert ends.tolist() == oracle.chunk_ends(oracle.config(2048, t), data).tolist()
    ends2, _ = eng.scan_batch(pg.make_config(2048), to_dev(torch, data), [0], [len(data)])   # table switch back
    assert ends2.tolist() == oracle.chunk_ends(oracle.config(2048), data).tolist()


def test_sha256_batch_all_small_lengths_and_alignments(eng, torch):
    data = rnd(70_000, 21)
    offs, lens = [], []
    for n in list(range(0, 200)) + [255, 256, 257, 1000, 4096, 65_535]:
        for a in (0, 1, 2, 3, 5, 13):
            offs.append(a + 7 * (n % 11))
            lens.append(n)
    # the last input is a host base with every range empty at offset 0: nothing is staged and the base is not read
    for host, offs, lens in ((False, offs, lens), (True, offs, lens), (True, [0] * 4, [0] * 4)):
        dig = eng.sha256_batch(data if host else to_dev(torch, data), offs, lens)
        for o, n, d in zip(offs, lens, dig, strict=True):
            assert bytes(d) == hashlib.sha256(data[o:o + n].tobytes()).digest(), (o, n, host)


@pytest.mark.parametrize("variant", [0, 1])
def test_chunk_digest_batch_matches_oracle(eng, torch, variant):
    eng.set_kernel_variant(variant)
    try:
        arrs = [rnd(n, 300 + i) for i, n in enumerate([0, 5, 70_000, 1, 333_333, 64, 1 << 20])]
        buf, off, ln = pack(arrs, align=1, lead=3)
        for avg in (256, 4096):
            rec = eng.chunk_digest_batch(pg.make_config(avg), to_dev(torch, buf), off, ln)
            ref = oracle.chunk_digest_streams(oracle.config(avg), arrs, threads=4)
            assert rec.tobytes() == ref.tobytes()
    finally:
        eng.set_kernel_variant(0)


def test_golden_vectors_through_the_c_abi(eng, torch):
    for ln in (GOLDEN / "chunks_oracle.jsonl").read_text().splitlines():
        g = json.loads(ln)
        c = pg.corpus(seed=g["seed"], file_len=g["len"], block_len=g["block_len"])
        stride = (g["len"] + 255) // 256 * 256
        dev = torch.zeros(stride * (g["file_id"] + 1), dtype=torch.uint8, device="cuda")
        eng.corpus_fill(c, 0, g["file_id"] + 1, dev, stride)
        rec = eng.chunk_digest_batch(pg.make_config(g["avg"]), dev, [g["file_id"] * stride], [g["len"]])
        assert rec["end_off"].tolist() == g["cuts"]
        assert [bytes(x).hex() for x in rec["digest"]] == g["digests"]


@pytest.mark.parametrize("kw", [dict(), dict(dup_permille=300, run_blocks=2), dict(edit_mode=1),
                                dict(edit_mode=2, dup_permille=300, run_blocks=3)])
def test_device_corpus_equals_oracle_corpus(eng, torch, kw):
    for file_len, block_len in ((1 << 16, 1 << 12), (100_003, 4096), (7, 8), (8192, 8192)):
        co = oracle.corpus(seed=2, file_len=file_len, block_len=block_len, **kw)
        cg = pg.corpus(seed=2, file_len=file_len, block_len=block_len, **kw)
        stride = (file_len + 255) // 256 * 256
        dev = torch.zeros(stride * 5, dtype=torch.uint8, device="cuda")
        eng.corpus_fill(cg, 3, 5, dev, stride)
        host = dev.cpu().numpy().reshape(5, stride)
        for i in range(5):
            assert (host[i, :file_len] == oracle.corpus_file(co, 3 + i)).all(), (kw, file_len, i)


def test_cfg2_shape_scaled_parity_and_invariants(eng, torch):
    """BASELINE cfg2 shape (N x 64 MiB files, 4 MiB average) scaled to 12 files: cut-for-cut and
    digest-for-digest against the oracle; plus the size-independent invariants."""
    n_files, file_len = 12, 64 << 20
    cg = pg.corpus(seed=2, file_len=file_len)
    dev = torch.empty(n_files * file_len, dtype=torch.uint8, device="cuda")
    eng.corpus_fill(cg, 0, n_files, dev, file_len)
    off = np.arange(n_files, dtype=np.uint64) * file_len
    ln = np.full(n_files, file_len, dtype=np.uint64)
    cfg = pg.buzhash.NewConfig(4096)
    rec = eng.chunk_digest_batch(cfg, dev, off, ln)
    files = oracle.corpus_files(oracle.corpus(seed=2, file_len=file_len), 0, n_files)
    ref = oracle.chunk_digest_streams(oracle.config(4 << 20), files, threads=os.cpu_count())
    assert rec.tobytes() == ref.tobytes()
    for s in range(n_files):
        e = np.concatenate([[0], rec[rec["stream"] == s]["end_off"]]).astype(np.int64)
        lens = np.diff(e)
        assert e[-1] == file_len and (lens[:-1] >= cfg.min).all() and (lens <= cfg.max).all()


def test_incremental_edits_resynchronise_like_the_oracle(eng, torch):
    """BASELINE cfg5: same corpus with ~1 % byte edits (uniform) and with one edited byte in ~1 % of
    blocks (clustered): boundaries shift exactly as the oracle's do, and away from the edits
    the chunks (digests) are unchanged."""
    n_files, file_len, bl = 6, 8 << 20, 1 << 16
    cfg_g, cfg_o = pg.make_config(1 << 16), oracle.config(1 << 16)
    off = np.arange(n_files, dtype=np.uint64) * file_len
    ln = np.full(n_files, file_len, dtype=np.uint64)
    results = {}
    for mode in (0, 1, 2):
        cg = pg.corpus(seed=5, file_len=file_len, block_len=bl, edit_mode=mode)
        dev = torch.empty(n_files * file_len, dtype=torch.uint8, device="cuda")
        eng.corpus_fill(cg, 0, n_files, dev, file_len)
        rec = eng.chunk_digest_batch(cfg_g, dev, off, ln)
        files = oracle.corpus_files(oracle.corpus(seed=5, file_len=file_len, block_len=bl, edit_mode=mode), 0, n_files)
        assert rec.tobytes() == oracle.chunk_digest_streams(cfg_o, files, threads=4).tobytes(), mode
        results[mode] = {bytes(d) for d in rec["digest"]}
    assert len(results[0] & results[2]) > 0.5 * len(results[0])      # clustered edits: most chunks survive
    assert len(results[0] & results[1]) < 0.05 * len(results[0])     # uniform 1 % edits: nothing survives


def test_async_jobs_overlap_and_match_sync(eng, torch):
    cfg = pg.make_config(1 << 16)
    devs, jobs = [], []
    for k in range(5):
        data = rnd(6 << 20, 400 + k)
        d = to_dev(torch, data)
        devs.append((d, data))
        jobs.append(eng.submit(cfg, d, [0, 3 << 20], [3 << 20, 3 << 20]))
    for (d, data), j in zip(devs, jobs):
        rec, timing = j.wait()
        ref = oracle.chunk_digest_streams(oracle.config(1 << 16), [data[:3 << 20], data[3 << 20:]])
        assert rec.tobytes() == ref.tobytes() and timing["chunks"] == len(ref)


def test_host_input_is_staged_in_groups(torch):
    os.environ["PBSGPU_STAGE_BYTES"] = str(1 << 20)      # force several staging groups
    try:
        e = pg.Engine(0)
    finally:
        del os.environ["PBSGPU_STAGE_BYTES"]
    try:
        arrs = [rnd(n, 500 + i) for i, n in enumerate([400_000, 0, 900_000, 1_500_000, 10, 700_000, 333])]
        rec = e.chunk_digest_streams(pg.make_config(4096), arrs)
        assert rec.tobytes() == oracle.chunk_digest_streams(oracle.config(4096), arrs).tobytes()
        pinned = e.host_alloc(2_000_000)                 # C-owned pinned staging, as the Go side would use
        pinned[:] = rnd(2_000_000, 77)
        rec = e.chunk_digest_batch(pg.make_config(4096), pinned, [0, 1_000_000], [1_000_000, 1_000_000])
        ref = oracle.chunk_digest_streams(oracle.config(4096), [np.array(pinned[:1_000_000]), np.array(pinned[1_000_000:])])
        assert rec.tobytes() == ref.tobytes()
        e.host_free(pinned)
    finally:
        e.close()


def test_output_capacity_error_reports_needed(eng, torch):
    import ctypes as C
    data = rnd(100_000, 1)
    cfg = pg.make_config(256)
    off = np.array([0], dtype=np.uint64); ln = np.array([len(data)], dtype=np.uint64)
    out = np.zeros(3, dtype=pg.CHUNK_DTYPE); n_out = C.c_uint64()
    d = to_dev(torch, data)
    rc = eng._L.pbsgpu_chunk_digest_batch(eng._h, C.byref(cfg), d.data_ptr(), off.ctypes.data, ln.ctypes.data, 1, None,
                                          out.ctypes.data, 3, C.byref(n_out))
    assert rc == -34 and n_out.value == len(oracle.chunk_ends(oracle.config(256), data))
    assert b"capacity" in eng._L.pbsgpu_strerror(eng._h)


# ---- a4: digest set ---------------------------------------------------------------
def test_digest_set_matches_oracle_set(eng):
    rng = np.random.default_rng(12)
    s_g, s_o = eng.digest_set(16), oracle.DigestSet(16)
    pool = rng.integers(0, 256, size=(5000, 32), dtype=np.uint8)
    for rnd_i in range(6):                                # growth + rehash happen along the way
        idx = rng.integers(0, 1000 * (rnd_i + 1), size=3000).clip(max=4999)
        batch = pool[idx]
        assert (s_g.insert(batch) == s_o.probe(batch, insert=True)).all()
        assert len(s_g) == len(s_o)
        probe = pool[rng.integers(0, 5000, size=2000)]
        assert (s_g.probe(probe) == s_o.probe(probe, insert=False)).all()
        assert len(s_g) == len(s_o)


def test_digest_set_tag_collisions_and_identical_runs(eng):
    """Digests that share their first 8 bytes (the table's tag) but differ later must stay
    distinct; a run of identical digests (e.g. zero-filled files) is one entry."""
    s = eng.digest_set(4)
    d = np.zeros((300, 32), dtype=np.uint8)
    d[:, :8] = 7                                          # identical tag
    d[:100, 31] = np.arange(100)                          # 100 distinct digests
    d[100:200, 31] = np.arange(100)                       # the same 100 again
    d[200:, 31] = 5                                       # 100 copies of one of them
    hit = s.insert(d)
    assert hit[:100].sum() == 0 and hit[100:].all() and len(s) == 100
    z = np.zeros((1, 32), dtype=np.uint8)                 # all-zero digest: tag 0 is remapped, still exact
    assert s.insert(z)[0] == 0 and s.probe(z)[0] == 1 and len(s) == 101


def test_batch_with_set_flags_known_chunks_in_order(eng, torch):
    """30 %-duplicate corpus (BASELINE cfg3 shape, scaled): the KNOWN flags and the hit-rate equal
    what the oracle computes in (file, chunk) order; a second pass over the same data is 100 % known."""
    n_files, file_len, bl = 24, 4 << 20, 1 << 16
    kw = dict(seed=3, file_len=file_len, block_len=bl, run_blocks=8, dup_permille=300)
    dev = torch.empty(n_files * file_len, dtype=torch.uint8, device="cuda")
    eng.corpus_fill(pg.corpus(**kw), 0, n_files, dev, file_len)
    off = np.arange(n_files, dtype=np.uint64) * file_len
    ln = np.full(n_files, file_len, dtype=np.uint64)
    s = eng.digest_set()
    rec = eng.chunk_digest_batch(pg.make_config(1 << 14), dev, off, ln, s)
    files = oracle.corpus_files(oracle.corpus(**kw), 0, n_files)
    ref = oracle.chunk_digest_streams(oracle.config(1 << 14), files, threads=4)
    so = oracle.DigestSet()
    ref["flags"] = so.probe(ref["digest"], insert=True)
    assert rec.tobytes() == ref.tobytes()
    hit_rate = (rec["flags"] & 1).mean()
    assert 0.15 < hit_rate < 0.40, hit_rate
    rec2 = eng.chunk_digest_batch(pg.make_config(1 << 14), dev, off, ln, s)
    assert (rec2["flags"] & 1).all() and len(s) == len(so)


def test_seed_from_previous_dynamic_index(eng, torch):
    data = rnd(3_000_000, 31)
    cfg = pg.make_config(1 << 14)
    rec = eng.chunk_digest_batch(cfg, to_dev(torch, data), [0], [len(data)])
    didx = bytearray(4096)                                           # header (magic/uuid/ctime/csum: not read)
    for r in rec[: len(rec) // 2]:                                   # previous snapshot held the first half
        didx += int(r["end_off"]).to_bytes(8, "little") + bytes(r["digest"])
    s = eng.digest_set()
    assert s.seed_didx(bytes(didx)) == len(rec) // 2
    rec2 = eng.chunk_digest_batch(cfg, to_dev(torch, data), [0], [len(data)], s)
    assert (rec2["flags"][: len(rec) // 2] & 1).all() and not (rec2["flags"][len(rec) // 2:] & 1).any()
    with pytest.raises(pg.PbsGpuError):
        s.seed_didx(b"\0" * 4097)


# ---- streaming form ---------------------------------------------------------------------
@pytest.mark.parametrize("window", [4096, 20_000, 1 << 20])
def test_streaming_is_split_invariant(torch, window):
    os.environ["PBSGPU_STREAM_WINDOW"] = str(window)
    e = pg.Engine(0)
    try:
        data = rnd(700_001, 41)
        ref = oracle.chunk_digest(oracle.config(1024), data)
        for pieces in ([len(data)], [1, 63, 64, 1000, 99_999, 10**9], [7777] * 200):
            st = e.stream(pg.make_config(1024))
            pos, got = 0, []
            for p in pieces:
                if pos >= len(data):
                    break
                st.write(data[pos:pos + p]); pos += p
                got.append(st.poll())
            got.append(st.finish())
            rec = np.concatenate(got)
            assert rec.tobytes() == ref.tobytes(), (window, pieces[:3])
            with pytest.raises(pg.PbsGpuError):
                st.write(b"x")
            st.close()
        st = e.stream(pg.make_config(1024))                          # empty stream: no chunks
        assert len(st.finish()) == 0
    finally:
        del os.environ["PBSGPU_STREAM_WINDOW"]
        e.close()


# ---- reference-facing mirror -----------------------------------------------------------
def test_dedup_writer_mirror_of_the_reference_surface(eng):
    import io
    cfg = pg.buzhash.NewConfigBytes(4096)
    uploaded = {}
    w = pg.transfer.NewRemoteDedupSplitArchiveWriter(eng, cfg, known=eng.digest_set(),
                                                     upload=lambda d, b: uploaded.__setitem__(d, b))
    files = {"a.bin": rnd(200_000, 51), "b.bin": rnd(50_000, 52), "empty": rnd(0, 53)}
    files["a-copy.bin"] = files["a.bin"].copy()
    for name, data in files.items():
        w.WriteEntryReader(pg.transfer.Entry(name, len(data)), io.BytesIO(data.tobytes()), len(data))
    with pytest.raises(IOError):                                     # io.ReadFull semantics: short reader is an error
        w.WriteEntryReader(pg.transfer.Entry("short", 10), io.BytesIO(b"abc"), 10)
    index = w.Finish()
    ref = oracle.chunk_digest_streams(oracle.config(4096), list(files.values()))
    assert [(r.end_off, r.digest) for r in index] == [(int(r["end_off"]), bytes(r["digest"])) for r in ref]
    known = [r.known for r in index]
    n_a = sum(1 for r in index if r.path == "a.bin")
    assert not any(known[:n_a]) and all(r.known for r in index if r.path == "a-copy.bin")
    for d, b in uploaded.items():
        assert hashlib.sha256(b).digest() == d
    assert len(uploaded) == len({r.digest for r in index})
    assert w.backed_hashes == {k: _xxh3_ref(v) for k, v in files.items()}      # commit.go:725 ow.backedHashes


def test_cxx_host_mirror_driver(tmp_path):
    """The C++ mirror of the Go surface (include/pbsgpu.hpp) driving the C ABI from a non-Python
    process, with pinned staging filled by the caller -- what the cgo shim does."""
    import subprocess
    drv = Path(__file__).parent / "cxx" / "driver.bin"
    if not drv.exists():
        pytest.skip("driver not built (run __graft_entry__.build())")
    datas = {"f0.bin": rnd(3_000_000, 61), "f1.bin": rnd(10, 62), "f2.bin": rnd(0, 63), "f3.bin": rnd(777_777, 64)}
    paths = []
    for k, v in datas.items():
        (tmp_path / k).write_bytes(v.tobytes())
        paths.append(str(tmp_path / k))
    out = subprocess.run([str(drv), "16", *paths], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    assert lines[-1] == "config-error -22"
    ref = oracle.chunk_digest_streams(oracle.config(16 << 10), list(datas.values()))
    pay = [l.split() for l in lines if l.startswith("payload ")]
    pay_off = {l.split()[1]: int(l.split()[2]) for l in lines if l.startswith("payload-offset ")}
    lines = [l for l in lines if not l.startswith("payload")]
    # the layout-faithful writer: the same files as ONE pxar payload stream with suggested boundaries at the file starts
    from pbs_plus_b200 import transfer as tr
    parts, pos, starts = [tr.PXAR_PAYLOAD_START_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little")], 16, []
    for v in datas.values():
        starts.append(pos); parts += [tr.payload_header(len(v)), v.tobytes()]; pos += 16 + len(v)
    parts.append(tr.PXAR_PAYLOAD_TAIL_MARKER.to_bytes(8, "little") + (16).to_bytes(8, "little"))
    stream = np.frombuffer(b"".join(parts), dtype=np.uint8)
    pref = oracle.chunk_digest_forced(oracle.config(16 << 10), stream, np.array(starts, np.uint64))
    assert [(int(r[1]), r[2]) for r in pay] == [(int(r["end_off"]), bytes(r["digest"]).hex()) for r in pref]
    assert pay_off == dict(zip(paths, starts))
    rows = [l.split() for l in lines[:-1] if not l.startswith("xxh3 ")]
    xx = {l.split()[1]: int(l.split()[2], 16) for l in lines if l.startswith("xxh3 ")}
    assert xx == {p: _xxh3_ref(v) for p, v in zip(paths, datas.values())}      # backedHashes mirror (commit.go:725)
    for ps in (0, 1):
        got = [(r[1], int(r[2]), r[3], int(r[4])) for r in rows if int(r[0]) == ps]
        assert [(g[1], g[2]) for g in got] == [(int(r["end_off"]), bytes(r["digest"]).hex()) for r in ref]
        assert all(g[3] == ps for g in got)          # first pass: all new; second pass: all known


def test_empty_batch_and_many_tiny_streams(eng, torch):
    cfg = pg.make_config(256)
    assert len(eng.chunk_digest_batch(cfg, torch.zeros(16, dtype=torch.uint8, device="cuda"), [], [])) == 0
    rng = np.random.default_rng(71)
    arrs = [rnd(int(n), 1000 + i) for i, n in enumerate(rng.integers(0, 700, size=3000))]
    buf, off, ln = pack(arrs, align=16)
    rec = eng.chunk_digest_batch(cfg, to_dev(torch, buf), off, ln)
    ref = oracle.chunk_digest_streams(oracle.config(256), arrs, threads=4)
    assert rec.tobytes() == ref.tobytes()


def test_partition_info_is_consistent(eng, torch):
    long_sms, bulk_sms = eng.partition_info()
    total = eng.device_info()["sm_count"]
    scan_sms = eng.scan_partition_sms()
    chip = torch.cuda.get_device_properties(eng.device).multi_processor_count
    assert (long_sms, bulk_sms) == (0, 0) or (long_sms >= 8 and long_sms + bulk_sms + scan_sms <= chip and bulk_sms == total)
    assert scan_sms == 0 or scan_sms >= 8


def test_all_long_chunks_take_the_latency_kernel(eng, torch):
    """Constant data => every chunk is a forced cut at max (> 2.5 x avg): the whole batch goes through the
    long-chunk (split) kernel when the hybrid launch is active; digests must still match."""
    data = np.zeros(3_000_000, dtype=np.uint8)
    data[::4099] = 7
    for avg in (4096, 65536):
        rec = eng.chunk_digest_batch(pg.make_config(avg), to_dev(torch, data), [0, 1_000_001], [1_000_001, 1_999_999])
        ref = oracle.chunk_digest_streams(oracle.config(avg), [data[:1_000_001], data[1_000_001:]])
        assert rec.tobytes() == ref.tobytes()


def test_didx_image_build_parse_and_seed(eng, torch):
    """f1: the dynamic-index image of a batch equals the oracle's (hashlib checksum), parses back, verifies,
    rejects corruption, and seeds the known set."""
    from oracle import pyref
    arrs = [rnd(400_000, 81), rnd(0, 82), rnd(123_456, 83)]
    buf, off, ln = pack(arrs)
    rec = eng.chunk_digest_batch(pg.make_config(4096), to_dev(torch, buf), off, ln)
    img = eng.didx_build(rec, uuid=bytes(range(16)), ctime=1_700_000_000)
    lens = []
    prev = {0: 0, 1: 0, 2: 0}
    for r in rec:
        lens.append(int(r["end_off"]) - prev[int(r["stream"])]); prev[int(r["stream"])] = int(r["end_off"])
    assert img == pyref.didx_build(lens, [bytes(d) for d in rec["digest"]], bytes(range(16)), 1_700_000_000)
    ends, dig = eng.didx_parse(img)
    assert ends.tolist() == np.cumsum(lens).tolist() and (dig == rec["digest"]).all()
    bad = bytearray(img); bad[4096 + 9] ^= 1
    with pytest.raises(pg.PbsGpuError):
        eng.didx_parse(bytes(bad))
    s = eng.digest_set()
    assert s.seed_didx(img) == len(rec) and s.probe(rec["digest"]).all()
    assert len(eng.didx_parse(eng.didx_build(rec[:0]))[0]) == 0


def test_crc32_batch_matches_zlib(eng, torch):
    """f3: DataBlob payload checksums.  zlib.crc32 is the (authoritative) oracle."""
    import zlib
    data = rnd(3_000_000, 91)
    offs, lens = [], []
    for n in [0, 1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 63, 143, 144, 145, 4095, 4096, 4097, 4607, 4608, 4609, 8191, 131071,
              131072, 131073, 262144, 589823, 589824, 589825, 1_000_003, 2_500_000]:
        for a in (0, 1, 2, 3, 15, 16, 17):
            offs.append(a); lens.append(n)
    # the first input is a host base with every range empty at offset 0: nothing is staged and the base is not read
    for host, offs, lens in ((True, [0] * 4, [0] * 4), (True, offs, lens), (False, offs, lens)):
        crc = eng.crc32_batch(data if host else to_dev(torch, data), offs, lens)
        for o, n, c in zip(offs, lens, crc, strict=True):
            assert int(c) == zlib.crc32(data[o:o + n].tobytes()), (o, n, host)
    hdr = eng.blob_header(int(crc[-1]))
    assert hdr[:8] == bytes([66, 171, 56, 7, 190, 131, 112, 161]) and int.from_bytes(hdr[8:], "little") == int(crc[-1])


def test_cfg1_single_1gib_stream(eng, torch):
    """BASELINE config[0]: ONE 1 GiB synthetic stream, 4 MiB average -- the case the reference's CPU chunker
    runs.  Cut-for-cut and digest-for-digest against the oracle (single thread, SHA-NI)."""
    n = 1 << 30
    dev = torch.empty(n, dtype=torch.uint8, device="cuda")
    eng.corpus_fill(pg.corpus(seed=1, file_len=n), 0, 1, dev, n)
    rec = eng.chunk_digest_batch(pg.buzhash.NewConfig(4096), dev, [0], [n])
    ref = oracle.chunk_digest(oracle.config(4 << 20), oracle.corpus_file(oracle.corpus(seed=1, file_len=n), 0))
    assert rec.tobytes() == ref.tobytes() and 200 < len(rec) < 400 and int(rec["end_off"][-1]) == n
    # the same stream through the streaming form (state carried across 64 MiB writes)
    host = dev.cpu().numpy()
    st = eng.stream(pg.buzhash.NewConfig(4096))
    for i in range(0, n, 64 << 20):
        st.write(host[i:i + (64 << 20)])
    assert st.finish().tobytes() == ref.tobytes()
    st.close()


@pytest.mark.parametrize("env", [{"PBSGPU_PARTITION_SMS": "0"}, {"PBSGPU_PARTITION_SMS": "0", "PBSGPU_SHA_HYBRID": "2"},
                                 {"PBSGPU_PARTITION_SMS": "16"}])
def test_results_do_not_depend_on_the_sm_partition(torch, env):
    """No green contexts (fallback), forced hybrid launch without a partition, and another partition size:
    same chunks, same digests."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        e = pg.Engine(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    try:
        if env["PBSGPU_PARTITION_SMS"] == "0":
            assert e.partition_info() == (0, 0)
        arrs = [rnd(3_000_000, 700), rnd(10, 701), rnd(1_234_567, 702)]
        buf, off, ln = pack(arrs)
        rec = e.chunk_digest_batch(pg.make_config(1 << 16), to_dev(torch, buf), off, ln)
        assert rec.tobytes() == oracle.chunk_digest_streams(oracle.config(1 << 16), arrs).tobytes()
    finally:
        e.close()


def test_mostly_long_chunks_are_capped_for_the_latency_partition(eng, torch):
    """Zero-filled data cuts every chunk at max: far more 'long' chunks than the latency partition should take.
    The head is capped (longest first); results stay exact."""
    n = 96 << 20
    data = np.zeros(n, dtype=np.uint8)
    data[5::1_000_003] = 1
    rec = eng.chunk_digest_batch(pg.make_config(4096), to_dev(torch, data), [0], [n])     # 6144 chunks of 16 KiB
    assert len(rec) > 24 * 32 * 4
    assert rec.tobytes() == oracle.chunk_digest(oracle.config(4096), data).tobytes()


@pytest.mark.parametrize("variant", [0, 1])
def test_structured_data_kinds_match_oracle(eng, torch, variant):
    """Zeros, low-entropy, periodic and text-like data (where candidates are absent or dense and cuts are
    forced) through scan + SHA-256, both kernel variants."""
    eng.set_kernel_variant(variant)
    try:
        rng = np.random.default_rng(91)
        kinds = {
            "zeros": np.zeros(700_000, dtype=np.uint8),
            "ff": np.full(300_001, 255, dtype=np.uint8),
            "two-symbols": rng.integers(0, 2, size=500_000, dtype=np.uint8),
            "three-symbols": rng.integers(0, 3, size=500_003, dtype=np.uint8),
            "period-7": np.resize(rng.integers(0, 256, size=7, dtype=np.uint8), 400_000),
            "period-64": np.resize(rng.integers(0, 256, size=64, dtype=np.uint8), 400_000),
            "period-1000": np.resize(rng.integers(0, 256, size=1000, dtype=np.uint8), 600_000),
            "text": np.frombuffer((b"the quick brown fox jumps over the lazy dog\n" * 20000)[:777_777], dtype=np.uint8).copy(),
            "ramp": (np.arange(650_000) % 251).astype(np.uint8),
        }
        arrs = list(kinds.values())
        buf, off, ln = pack(arrs, align=16, lead=16)
        for avg in (256, 4096, 65536):
            rec = eng.chunk_digest_batch(pg.make_config(avg), to_dev(torch, buf), off, ln)
            ref = oracle.chunk_digest_streams(oracle.config(avg), arrs, threads=4)
            assert rec.tobytes() == ref.tobytes(), (avg, variant)
    finally:
        eng.set_kernel_variant(0)


# ---- K1 variant: lane-contiguous scan kernel (PBSGPU_SCAN_LANES=1, off by default) ---------------------------------
def _engine_with_env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return pg.Engine(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def test_scan_lanes_variant_matches_oracle(torch):
    """k_scan_lanes (64 KiB super-tiles, per-lane TMA pieces) must give the boundaries k_scan_tuned gives: streams
    with several super-tiles, tails, a stream below one super-tile, misaligned streams (plain-tile path only)."""
    e = _engine_with_env({"PBSGPU_SCAN_LANES": "1"})
    try:
        arrs = [rnd(n, 900 + i) for i, n in enumerate([65536 * 5 + 777, 65536, 65535, 65537, 3 * 65536 + 8704, 100, 0,
                                                       1_000_003, 65536 * 2])]
        for avg in (256, 4096, 1 << 16):
            cfg_o = oracle.config(avg)
            want, want_first = oracle_ends(cfg_o, arrs)
            for align, lead in ((256, 0), (1, 3), (16, 16)):
                buf, off, ln = pack(arrs, align=align, lead=lead)
                ends, first = e.scan_batch(pg.make_config(avg), to_dev(torch, buf), off, ln)
                assert ends.tolist() == want and first.tolist() == want_first, (avg, align, lead)
        big = rnd(40_000_000, 950)
        rec = e.chunk_digest_batch(pg.make_config(1 << 16), to_dev(torch, big), [0], [len(big)])
        assert rec.tobytes() == oracle.chunk_digest(oracle.config(1 << 16), big).tobytes()
    finally:
        e.close()


# ---- f2: XXH3-64 of the commit walk (K7) ----------------------------------------------------------------------------
def _xxh3_ref(a):
    try:
        import xxhash                      # independent implementation (libxxhash binding)
        return xxhash.xxh3_64_intdigest(np.ascontiguousarray(a).tobytes())
    except ImportError:                    # the oracle restatement is pinned against it in the CPU suite
        return oracle.xxh3_64(a)


def test_xxh3_every_short_length_and_alignment(eng, torch):
    data = rnd(4096, 1200)
    lens = list(range(0, 1300)) + [2047, 2048, 2049, 3072, 3073, 4000]
    for lead in (0, 1, 5, 16):
        off = np.array([lead + (i % 7) for i in range(len(lens))], dtype=np.uint64)
        ln = np.array(lens, dtype=np.uint64)
        ok = off + ln <= len(data)
        off, ln2 = off[ok], ln[ok]
        want = np.array([_xxh3_ref(data[int(o): int(o + l)]) for o, l in zip(off, ln2)], dtype=np.uint64)
        got_dev = eng.xxh3_batch(to_dev(torch, data), off, ln2)
        got_host = eng.xxh3_batch(data, off, ln2)
        assert got_dev.tolist() == want.tolist(), lead
        assert got_host.tolist() == want.tolist(), lead
        assert [oracle.xxh3_64(data[int(o): int(o + l)]) for o, l in zip(off[:300], ln2[:300])] == want[:300].tolist()


def test_xxh3_long_streams_aligned_and_not(eng, torch):
    sizes = [1 << 20, (1 << 20) + 1, (1 << 20) - 1, 5_000_003, 64 * 1024, 1025, 1024, 241, 240, 0, 3 << 20, 777_777]
    arrs = [rnd(n, 1300 + i) for i, n in enumerate(sizes)]
    want = [_xxh3_ref(a) for a in arrs]
    for align, lead in ((256, 0), (1, 0), (1, 7), (16, 16)):
        buf, off, ln = pack(arrs, align=align, lead=lead)
        assert eng.xxh3_batch(to_dev(torch, buf), off, ln).tolist() == want, (align, lead)
    buf, off, ln = pack(arrs)
    assert eng.xxh3_batch(buf, off, ln).tolist() == want          # host base: staged by the library


def test_xxh3_is_pass_invariant(torch):
    """A tiny per-pass block budget forces many passes with carried chain state: same hashes."""
    e = _engine_with_env({"PBSGPU_XXH3_CAP_BLOCKS": "37"})
    try:
        sizes = [300_000, 5, 70_001, 1 << 20, 0, 2048, 123_456, 1025]
        arrs = [rnd(n, 1400 + i) for i, n in enumerate(sizes)]
        buf, off, ln = pack(arrs, align=16)
        assert e.xxh3_batch(to_dev(torch, buf), off, ln).tolist() == [_xxh3_ref(a) for a in arrs]
    finally:
        e.close()


def test_fused_batch_returns_chunks_and_file_xxh3(torch):
    """pbsgpu_chunk_digest_batch_xxh3: the chunk records of the plain call plus every stream's XXH3-64, from device
    input and from host input staged in several groups."""
    e = _engine_with_env({"PBSGPU_STAGE_BYTES": str(1 << 20)})
    try:
        arrs = [rnd(n, 1500 + i) for i, n in enumerate([400_000, 0, 900_000, 1_500_000, 10, 700_000, 333, 1024])]
        want_rec = oracle.chunk_digest_streams(oracle.config(4096), arrs).tobytes()
        want_h = [_xxh3_ref(a) for a in arrs]
        buf, off, ln = pack(arrs)
        cfg = pg.make_config(4096)
        rec, h = e.chunk_digest_batch_xxh3(cfg, buf, off, ln)                      # host base
        assert rec.tobytes() == want_rec and h.tolist() == want_h
        rec, h = e.chunk_digest_batch_xxh3(cfg, to_dev(torch, buf), off, ln)       # device base
        assert rec.tobytes() == want_rec and h.tolist() == want_h
        ds = e.digest_set()
        rec, h = e.chunk_digest_batch_xxh3(cfg, to_dev(torch, buf), off, ln, ds)   # with the known-set
        assert h.tolist() == want_h and len(ds) == len({bytes(r["digest"]) for r in rec})
    finally:
        e.close()


def test_xxh3_golden_vectors_through_the_c_abi(eng, torch):
    """K7 against the committed libxxhash vectors (independent of python-xxhash being installed on the box)."""
    recs = [json.loads(l) for l in (GOLDEN / "xxh3_libxxhash.jsonl").read_text().splitlines()]
    arrs, want = [], []
    for r in recs:
        c = oracle.corpus(seed=r["seed"], file_len=max(r["len"] + r["lead"], 1), block_len=r["block_len"])
        arrs.append(oracle.corpus_file(c, 0)[r["lead"]: r["lead"] + r["len"]])
        want.append(int(r["xxh3_64"], 16))
    for align in (256, 1):
        buf, off, ln = pack(arrs, align=align)
        assert eng.xxh3_batch(to_dev(torch, buf), off, ln).tolist() == want, align


def test_verify_backed_file_hashes_on_the_gpu(eng, tmp_path):
    """The commit's second phase (commit.go:957-976) through the engine: hashes recorded by the fused batch call
    verify, a changed file is reported with the reference's message."""
    import io
    files = {"x.bin": rnd(500_000, 1601), "y.bin": rnd(77, 1602), "z.bin": rnd(0, 1603)}
    w = pg.transfer.DedupWriter(eng, pg.buzhash.NewConfigBytes(4096))
    for k, v in files.items():
        (tmp_path / k).write_bytes(v.tobytes())
        w.WriteEntryReader(pg.transfer.Entry(k, len(v)), io.BytesIO(v.tobytes()), len(v))
    w.Finish()
    opener = lambda rel: open(tmp_path / rel, "rb")
    pg.transfer.verifyBackedFileHashes(eng, opener, w.backed_hashes)
    raw = files["y.bin"].tobytes()
    (tmp_path / "y.bin").write_bytes(bytes([raw[0] ^ 0xFF]) + raw[1:])
    with pytest.raises(IOError, match='backed file "y.bin" content hash differs'):
        pg.transfer.verifyBackedFileHashes(eng, opener, w.backed_hashes)
