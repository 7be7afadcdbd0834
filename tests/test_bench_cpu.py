"""CPU-only checks of bench.py: the reference arm runs (it is the one bench leg that needs no GPU),
prints one well-formed JSON line, and the interval/traffic helpers behave."""
import importlib.util
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _bench():
    spec = importlib.util.spec_from_file_location("bench_mod", ROOT / "bench.py")
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_union_of_overlapping_kernel_intervals():
    b = _bench()
    assert b.union_ms([]) == 0
    assert b.union_ms([(0, 10), (5, 20), (30, 40)]) == 30
    assert b.union_ms([(3, 4), (0, 10)]) == 10


def test_instruction_ceiling_counts_every_sm():
    b = _bench()
    c = b.instr_ceiling(132, 1980.0, 500.0)      # H100 SXM: 132 SMs
    assert c["sm_count"] == 132 and 850 < c["alu_pipe_GBps"] < 900 and abs(c["frac_of_alu_pipe"] - 500.0 / c["alu_pipe_GBps"]) < 1e-9
    assert b.instr_ceiling(132, None, 1.0) is None


def test_dump_outputs_is_exact_small_and_reproducible(tmp_path):
    """--dump-outputs: every record while they fit, a fixed seeded sample once 64 MB (headers included) would be
    exceeded; the float64 arrays hold the record fields exactly."""
    import numpy as np
    sys.path.insert(0, str(ROOT))
    from pbs_plus_b200._lib import CHUNK_DTYPE
    b = _bench()
    rng = np.random.default_rng(5)
    for n in (10, 300_000):
        rec = np.zeros(n, CHUNK_DTYPE)
        rec["stream"] = rng.integers(0, 1024, n)
        rec["flags"] = rng.integers(0, 2, n)
        rec["end_off"] = rng.integers(0, 1 << 52, n)
        rec["digest"] = rng.integers(0, 256, (n, 32))
        dumps = []
        for run in ("a", "b"):
            b.dump_outputs(tmp_path / f"{n}{run}", rec)
            files = sorted((tmp_path / f"{n}{run}").glob("*.npy"))
            assert sum(f.stat().st_size for f in files) <= 64_000_000
            dumps.append({f.stem: np.load(f) for f in files})
        a = dumps[0]
        assert all(np.array_equal(a[k], dumps[1][k]) and a[k].dtype == np.float64 for k in a)
        rows = a["rows"].astype(np.int64)
        assert (len(rows) == n) == (n == 10) and (np.diff(rows) > 0).all()
        assert (a["end_off"] == rec["end_off"][rows]).all() and (a["digest"] == rec["digest"][rows]).all()
        assert (a["stream"] == rec["stream"][rows]).all() and (a["flags"] == rec["flags"][rows]).all()


def test_cfg4_expected_entries_are_found_by_shape(tmp_path, monkeypatch):
    b = _bench()
    (tmp_path / "profiles").mkdir()
    (tmp_path / "profiles" / "r02_cfg4_expected.json").write_text(json.dumps({"entries": [
        {"world": 2, "files_per_rank": 1024, "file_mib": 64, "chunks": 10, "known": 3}]}))
    monkeypatch.setattr(b, "ROOT", tmp_path)
    assert b.expected_cfg4_hits(2, 1024, 64)["known"] == 3
    assert b.expected_cfg4_hits(4, 1024, 64) is None


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
                          "--file-mib", "1"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "GiB/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_reference_arm_nonzero_rank_is_silent():
    import os
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                         capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""
