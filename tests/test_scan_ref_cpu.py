"""Pin tests/scan_ref.py (the candidate reference, the K2 restatement and candidate planting) against the oracle, on the
CPU.  The GPU scan-edge tests rely on each of these facts."""
import numpy as np
import pytest

import oracle
import scan_ref as sr


def _tables():
    rng = np.random.default_rng(11)
    return {"default": oracle.default_table(),
            "random1": rng.integers(0, 1 << 32, size=256, dtype=np.uint64).astype(np.uint32),
            "random2": rng.integers(0, 1 << 32, size=256, dtype=np.uint64).astype(np.uint32)}


@pytest.mark.parametrize("name", ["default", "random1", "random2"])
def test_candidates_match_the_oracle_window_hash(name):
    table = _tables()[name]
    rng = np.random.default_rng(5)
    data = rng.integers(0, 256, size=300_000, dtype=np.uint8)
    pos = np.concatenate([np.arange(63, 200), rng.integers(63, len(data), size=3000)])
    for mask in (511, 8191):
        got = set(sr.candidates(table, mask, data).tolist())
        for i in pos.tolist():
            h = oracle.window_hash(table, data[i - 63: i + 1])
            assert ((h & mask) >= mask - 2) == (i in got), (name, mask, i)
    # a sub-range gives the same positions as the whole stream, across block edges
    full = sr.candidates(table, 511, data)
    sub = sr.candidates(table, 511, data, 70_001, 290_000)
    assert sub.tolist() == full[(full >= 70_001) & (full < 290_000)].tolist()


@pytest.mark.parametrize("avg", [256, 512, 4096, 1 << 16, 1 << 22])
def test_resolve_matches_the_oracle_chunker(avg):
    n = 3_000_000 if avg >= 1 << 16 else 200_000
    data = np.random.default_rng(avg).integers(0, 256, size=n, dtype=np.uint8)
    cfg = oracle.config(avg)
    c = sr.candidates(oracle.default_table(), cfg.mask, data)
    assert sr.resolve(c, n, cfg) == oracle.chunk_ends(cfg, data).tolist()


def test_resolve_without_eof_leaves_the_undecided_tail():
    data = np.random.default_rng(8).integers(0, 256, size=100_000, dtype=np.uint8)
    cfg = oracle.config(1024)
    full = sr.resolve(sr.candidates(oracle.default_table(), cfg.mask, data), len(data), cfg)
    part = sr.resolve(sr.candidates(oracle.default_table(), cfg.mask, data), len(data), cfg, eof=False)
    assert part == full[:len(part)] and full[-1] - part[-1] <= cfg.max and len(full) - len(part) <= 1


@pytest.mark.parametrize("avg", [512, 4096, 1 << 16])
def test_resolve_with_forced_boundaries_matches_the_oracle(avg):
    rng = np.random.default_rng(avg + 1)
    n = 400_000
    data = rng.integers(0, 256, size=n, dtype=np.uint8)
    cfg = oracle.config(avg)
    c = sr.candidates(oracle.default_table(), cfg.mask, data)
    forced = sorted(set(rng.integers(1, n, size=60).tolist()) | {int(c[0]) + 1, int(c[5]) + 1, cfg.min})
    want = oracle.chunk_digest_forced(cfg, data, forced)["end_off"].tolist()
    assert sr.resolve(c, n, cfg, forced=forced) == want


@pytest.mark.parametrize("name", ["default", "random1", "random2"])
def test_zero_background_has_no_candidates(name):
    z = np.zeros(70_000, dtype=np.uint8)
    for mask in (511, 8191, (1 << 23) - 1):
        assert len(sr.candidates(_tables()[name], mask, z)) == 0


@pytest.mark.parametrize("avg", [256, 512, 4096, 1 << 16, 1 << 22, 1 << 29])
def test_found_patterns_give_one_candidate_wherever_they_are_placed(avg):
    table = sr.purpose_table(2 * avg - 1) if avg == 1 << 29 else oracle.default_table()
    pat = sr.find_pattern(table, 2 * avg - 1)
    assert pat.d in (32, 33)
    cfg = oracle.config(avg, table)
    rng = np.random.default_rng(avg)
    n = 20_000
    for p in [62, 63, 64, 65, 100, 271, 272, 1023, 1024, n - 1] + rng.integers(63, n, size=20).tolist():
        a = np.zeros(n, dtype=np.uint8)
        o = p - pat.d
        a[o: o + 3] = np.frombuffer(pat.bytes, dtype=np.uint8)
        assert sr.candidates(table, cfg.mask, a).tolist() == ([p] if p >= 63 else [])
        for i in (p, p - 1, p + 1):                     # the oracle's own window hash agrees
            if 63 <= i < n:
                h = oracle.window_hash(table, a[i - 63: i + 1])
                assert ((h & cfg.mask) >= cfg.break_min) == (i == p)


def test_plant_checks_every_position_and_the_oracle_cuts_there():
    cfg = oracle.config(512)
    pat = sr.find_pattern(oracle.default_table(), cfg.mask)
    pos = [62, 200, 500, 1000, 1127, 4000, 4999]
    a = sr.plant(5000, pos, pat)
    assert sr.candidates(pat.table, pat.mask, a).tolist() == pos[1:]
    assert oracle.chunk_ends(cfg, a).tolist() == sr.resolve(pos[1:], len(a), cfg)
    with pytest.raises(AssertionError):               # two patterns too close: their windows interfere or overlap
        sr.plant(5000, [300, 301], pat)
