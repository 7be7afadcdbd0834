"""Reference for the chunker's front half: K1's boundary candidates and K2's min/max rule, plus exact candidate planting.

  candidates   H(i) = rotl(Q[i] ^ Q[i-64], i mod 32), Q = XOR-prefix of rotr(T[b[p]], p mod 32) with Q[-k] = 0; this is
               the 64-byte buzhash window XOR_{j<64} rotl(T[b[i-j]], j mod 32).  Position i is a candidate when i >= 63 and
               (H(i) & mask) >= mask - 2.  Blocks of a few MiB keep the memory bounded on long streams.
  resolve      K2 (csrc/resolve.cu): the next cut after `start` is the first candidate p >= start + min_eff - 1 with
               p + 1 <= start + max, otherwise start + max; min_eff = max(min, 65).  At EOF the short tail is a chunk;
               without EOF the undecided tail is left.  A suggested boundary B enters as the key B - 1.
  planting     On an all-zero background every window hashes to 0 under any table (each rotation occurs twice in 64
               bytes), so no position is a candidate.  A short pattern's candidates then depend only on the offset from
               the pattern, so one pattern with exactly one candidate at offset d puts a candidate at any chosen P.
"""
from __future__ import annotations

from bisect import bisect_left

import numpy as np

WINDOW = 64
_BLOCK = 4 << 20


def _rotl(x: np.ndarray, r) -> np.ndarray:
    """rotl32 of u64-held u32 values; r scalar or array in [0, 32)."""
    r = np.asarray(r, dtype=np.uint64)
    return ((x << r) | (x >> (np.uint64(32) - r))) & np.uint64(0xFFFFFFFF)


def _rotr(x: np.ndarray, r) -> np.ndarray:
    r = np.asarray(r, dtype=np.uint64)
    return ((x >> r) | (x << (np.uint64(32) - r))) & np.uint64(0xFFFFFFFF)


def _hashes(table: np.ndarray, a: np.ndarray, base: int) -> np.ndarray:
    """H at positions base + 63 .. base + len(a) - 1 of a stream whose bytes base.. are `a` (len(a) >= 64)."""
    t = np.asarray(table, dtype=np.uint32).astype(np.uint64)
    p = (np.arange(len(a), dtype=np.uint64) + np.uint64(base)) % np.uint64(32)
    q = np.bitwise_xor.accumulate(_rotr(t[a], p))
    g = q[63:].copy()
    g[1:] ^= q[: len(a) - 64]
    return _rotl(g, p[63:])


def candidates(table, mask: int, data, lo: int = 0, hi: int | None = None) -> np.ndarray:
    """Candidate positions i in [lo, hi) of the stream `data` (sorted, int64)."""
    a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    hi = len(a) if hi is None else min(hi, len(a))
    lo = max(lo, 63)
    out = []
    m, thr = np.uint64(mask), np.uint64(mask - 2)
    for b0 in range(lo, hi, _BLOCK):
        b1 = min(b0 + _BLOCK, hi)
        h = _hashes(table, a[b0 - 63: b1], b0 - 63)
        out.append(np.nonzero((h & m) >= thr)[0] + b0)
    return np.concatenate(out).astype(np.int64) if out else np.zeros(0, dtype=np.int64)


def resolve(cands, n: int, cfg, eof: bool = True, forced=()) -> list[int]:
    """Chunk ends of one stream of n bytes from its candidate positions (and suggested boundaries)."""
    keys = sorted({int(c) for c in cands} | {int(b) - 1 for b in forced})
    min_eff, mx = max(int(cfg.min), 65), int(cfg.max)
    ends, start, k = [], 0, 0
    while start < n:
        k = bisect_left(keys, start + min_eff - 1, k)
        end = start + mx
        if k < len(keys) and keys[k] + 1 <= end:
            end = keys[k] + 1
        elif end > n:
            if not eof:
                break
            end = n
        ends.append(end)
        start = end
    return ends


class Pattern:
    """Bytes that, written at offset o of a zero background, make o + d the only candidate (under table and mask)."""

    def __init__(self, table, mask: int, data: bytes, d: int):
        self.table, self.mask, self.bytes, self.d = np.asarray(table, dtype=np.uint32), int(mask), bytes(data), int(d)

    @property
    def reach(self) -> int:
        """Positions o .. o + reach - 1 can hold a non-zero window hash."""
        return len(self.bytes) + WINDOW - 1


def pattern_candidates(table, mask: int, pat: bytes) -> list[int]:
    """Candidate offsets (relative to the pattern start) of `pat` on a zero background."""
    buf = np.zeros(WINDOW + len(pat) + WINDOW, dtype=np.uint8)
    buf[WINDOW: WINDOW + len(pat)] = np.frombuffer(pat, dtype=np.uint8)
    return [int(c) - WINDOW for c in candidates(table, mask, buf)]


def find_pattern(table, mask: int) -> Pattern:
    """The first 3-byte pattern (in order of d, then byte values) whose only candidate is at offset d = 32 or 33.

    For d in [2, 63] all three bytes are in the window: H(o + d) = rotl(X0, d) ^ rotl(X1, d - 1) ^ rotl(X2, d - 2)
    with Xm = T[b_m] ^ T[0].  Rotations are mod 32, so H(o + d) = H(o + d + 32) whenever both windows hold the whole
    pattern: only d = 32 and 33 (whose twins d - 32 do not) can be a single candidate.  The 2^24 triples are searched
    as 2^16 pairs against the 256 third terms."""
    t = np.asarray(table, dtype=np.uint32).astype(np.uint64)
    x = t ^ t[0]
    m = np.uint64(mask)
    for d in (32, 33):
        w = ((_rotl(x, d % 32)[:, None] ^ _rotl(x, (d - 1) % 32)[None, :]).reshape(-1)) & m
        r = _rotl(x, (d - 2) % 32) & m
        by_val: dict[int, list[int]] = {}
        for b2, v in enumerate(r.tolist()):
            by_val.setdefault(v, []).append(b2)
        rv = np.array(sorted(by_val), dtype=np.uint64)
        for tgt in (mask, mask - 1, mask - 2):
            want = w ^ np.uint64(tgt)
            for i in np.nonzero(np.isin(want, rv))[0].tolist():
                for b2 in by_val[int(want[i])]:
                    pat = bytes([i >> 8, i & 255, b2])
                    if pattern_candidates(table, mask, pat) == [d]:
                        return Pattern(table, mask, pat, d)
    raise LookupError(f"no 3-byte pattern with one candidate for mask {mask:#x}")


def purpose_table(mask: int, seed: int = 29) -> np.ndarray:
    """A random table whose bytes 1, 2, 3 hash to mask - 2 at offset 32 (for masks too wide for a search of the default
    table to be sure of a hit, such as the 2^30 - 1 of an average of 2^29): X0 ^ rotl(X1, 31) ^ rotl(X2, 30) = mask - 2.
    Not `mask` itself: H(o + 33) = rotl(H(o + 32), 1) would then be mask - 1, a second candidate."""
    t = np.random.default_rng(seed).integers(0, 1 << 32, size=256, dtype=np.uint64)
    x = t ^ t[0]
    x2 = _rotl(np.uint64(mask - 2) ^ x[1:2] ^ _rotl(x[2:3], 31), 2)[0]
    t[3] = x2 ^ t[0]
    return t.astype(np.uint32)


def offsets_for(positions, pat: Pattern) -> list[int]:
    """Pattern start for each wanted candidate position."""
    out = [int(p) - pat.d for p in positions]
    assert all(o >= 0 for o in out), "a planted candidate needs its pattern inside the stream"
    return out


def expected_candidates(positions) -> list[int]:
    """The positions a kernel must report for these planted ones: those with a whole window in the stream (>= 63)."""
    return sorted(int(p) for p in positions if int(p) >= 63)


def check_planted(get, n: int, positions, pat: Pattern) -> list[int]:
    """Assert that the stream of n bytes, zero outside the planted patterns, has exactly the expected candidates.

    `get(lo, hi)` returns the stream's bytes [lo, hi).  Only windows that reach a pattern are evaluated: every other
    window is all zero and hashes to 0, which is never a candidate (mask - 2 > 0)."""
    want = expected_candidates(positions)
    spans = sorted((o, min(n, o + pat.reach)) for o in offsets_for(positions, pat))
    merged: list[list[int]] = []
    for a, b in spans:
        if merged and a <= merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], b)
        else:
            merged.append([a, b])
    got = []
    for a, b in merged:
        lo = max(0, a - 63)
        got += (candidates(pat.table, pat.mask, get(lo, b)) + lo).tolist()
    got = sorted(c for c in got if c >= 63)
    assert got == want, f"planted {sorted(positions)} but the reference finds {got}"
    return want


def plant(n: int, positions, pat: Pattern) -> np.ndarray:
    """A stream of n bytes with the pattern's candidate at each position (asserted with `candidates`)."""
    a = np.zeros(n, dtype=np.uint8)
    pb = np.frombuffer(pat.bytes, dtype=np.uint8)
    for o in offsets_for(positions, pat):
        assert o + len(pb) <= n, f"pattern at {o} does not fit in {n} bytes"
        assert not a[o: o + len(pb)].any(), f"patterns overlap at {o}"
        a[o: o + len(pb)] = pb
    check_planted(lambda lo, hi: a[lo:hi], n, positions, pat)
    return a
