"""K1's three boundary-scan kernels and K2's min/max rule, candidate for candidate, at every index edge they have.

On a zero background no position is a candidate, and one short pattern (tests/scan_ref.py) puts exactly one candidate
wherever it is written, so every stream below holds exactly the candidates it was built with (asserted on the CPU
before it is used).  For each kernel, configuration and stream layout:
  * scan_batch's ends and stream_first equal the K2 restatement applied to the planted candidates;
  * the job reports exactly as many K1 candidates as were planted (Timing "candidates"): this sees a missed or extra
    candidate in the first min_eff - 1 bytes of a chunk, which no cut list shows;
  * the chunk records (stream, end, SHA-256) equal hashlib's digests of the expected chunks.
Kernels: k_scan_simple (variant 1), k_scan_tuned (default) and k_scan_lanes (PBSGPU_SCAN_LANES=1).  Stream offsets
that are 128 B aligned, 16 B but not 128 B aligned, and odd route to super-tiles, plain TMA tiles and the generic copy.
"""
import contextlib
import hashlib
import os

import numpy as np
import pytest

import oracle
import pbs_plus_b200 as pg
import scan_ref as sr

pytestmark = pytest.mark.gpu

TILE, LANE, SPAN, SUPER, PIECE, LANE_R = 8704, 272, 1024, 65536, 256, 2048
AVGS = [256, 512, 4096, 1 << 16, 1 << 22]
KERNELS = ["simple", "tuned", "lanes"]
LAYOUTS = {"aligned128": 0, "aligned16": 16, "odd": 1}    # lead of the first stream; every stride is a multiple of 128


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


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


@pytest.fixture(scope="module")
def engines():
    e, lanes = pg.Engine(0), _engine_with_env({"PBSGPU_SCAN_LANES": "1"})
    yield {"simple": (e, 1), "tuned": (e, 0), "lanes": (lanes, 0)}
    e.close()
    lanes.close()


@contextlib.contextmanager
def _kernel(engines, name):
    e, v = engines[name]
    e.set_kernel_variant(v)
    try:
        yield e
    finally:
        e.set_kernel_variant(0)


_PATTERNS = {}


def _pattern(avg):
    if avg not in _PATTERNS:
        table = sr.purpose_table(2 * avg - 1) if avg == 1 << 29 else pg.default_table()
        _PATTERNS[avg] = sr.find_pattern(table, 2 * avg - 1)
    return _PATTERNS[avg]


def _cfg(avg):
    return pg.make_config(avg, _pattern(avg).table if avg == 1 << 29 else None)


# ---- streams ----------------------------------------------------------------------------------------------------------
def _kernel_edge_streams():
    """(edge class, length, planted positions): one candidate per stream unless the class says otherwise."""
    S = []

    def add(cls, n, *pos):
        S.append((cls, n, list(pos)))
    for n in (3000, SUPER + 500):                            # in a plain tile, and in k_scan_lanes' first super-tile
        for p in (62, 63, 64):                               # 62: a hash hit no kernel may report; 63: first whole window
            add("first-window", n, p)
    for n in (96, 1000, TILE + 100, SUPER + 4097, 3 * SUPER):   # a candidate on the stream's last byte
        add("last-byte", n, n - 1)
    for k in (1, 2, 5):                                      # k_scan_simple: 1024-byte spans
        add("span-end", 8000, SPAN * k - 1)
        add("span-start", 8000, SPAN * k)
    for t in (0, 1):                                         # k_scan_tuned: first and last byte of lanes 0, 1, 30, 31
        for m in (0, 1, 30, 31):
            b = TILE * t + LANE * m
            if b >= 62:
                add("lane-first", 2 * TILE + 500, b)
            add("lane-last", 2 * TILE + 500, b + LANE - 1)
    for k in (1, 2):                                         # tile edges; at 8704k + 62 the window straddles the halo
        add("tile-last", 3 * TILE + 1000, TILE * k - 1)
        add("tile-first", 3 * TILE + 1000, TILE * k)
        add("tile-halo", 3 * TILE + 1000, TILE * k + 62)
    for k in (1, 2):                                         # partial last tiles: candidate on their last valid byte
        for v in (1, 271, 272, 273, 8703):
            add(f"partial-tile-{v}", TILE * k + v, TILE * k + v - 1)
    for L in (0, 5):                                         # k_scan_lanes: 256-byte piece edges inside a lane
        for s in (1, 2, 7):
            add("piece-last", 2 * SUPER + 300, LANE_R * L + PIECE * s - 1)
            add("piece-first", 2 * SUPER + 300, LANE_R * L + PIECE * s)
    for L in (1, 16, 31):                                    # lane edges inside a super-tile
        add("lane-r-last", 2 * SUPER + 300, SUPER + LANE_R * L - 1)
        add("lane-r-first", 2 * SUPER + 300, LANE_R * L)
    for u in (1, 2):                                         # super-tile edges
        add("super-last", 3 * SUPER + 100, SUPER * u - 1)
        add("super-first", 3 * SUPER + 100, SUPER * u)
    for n in (SUPER + 9000, 2 * SUPER + 70, 2 * SUPER + TILE + 5):   # last super-tile byte / first plain-tile byte
        f = n // SUPER * SUPER
        add("super-to-plain-last", n, f - 1)
        if f + 1 < n:
            add("super-to-plain-first", n, f)
        if f + TILE < n:
            add("plain-after-super", n, f + TILE - 1)
            add("plain-after-super", n, f + TILE)
    # 18 steps: every step index is a warp split point (the grid has at least ceil(18 / 8) CTAs of 8 warps), so splits
    # fall inside both super-tiles and round_unit moves them back; a candidate in every step of three lanes
    n = 2 * SUPER + TILE + 5
    add("warp-split", n, *[SUPER * u + LANE_R * L + PIECE * k + 100 for u in (0, 1) for L in (0, 17, 31) for k in range(8)],
        2 * SUPER + 1000, n - 1)
    return S


KERNEL_EDGE_CLASSES = {
    "every": {"first-window", "last-byte"},
    "simple": {"span-end", "span-start"},
    "tuned": {"lane-first", "lane-last", "tile-last", "tile-first", "tile-halo"} |
             {f"partial-tile-{v}" for v in (1, 271, 272, 273, 8703)},
    "lanes": {"piece-last", "piece-first", "lane-r-last", "lane-r-first", "super-last", "super-first",
              "super-to-plain-last", "super-to-plain-first", "plain-after-super", "warp-split"},
}


def _rule_edge_streams(avg):
    """Min/max rule edges of one configuration, relative to a chunk start."""
    cfg = _cfg(avg)
    min_eff, mx = max(int(cfg.min), 65), int(cfg.max)
    f = min_eff - 1                                          # first_ok of the chunk starting at 0
    S = [("first_ok-1", mx + 500, [f - 1]),                  # skipped: the chunk is cut at max
         ("first_ok", mx + 500, [f]),
         # cuts at max by the candidate, where the max rule cuts too: K2's `pos + 1 <= end` and `pos + 1 < end` give
         # the same cut here (and everywhere, since pos < len), so no cut list can tell them apart
         ("max-1", 2 * mx + 100, [mx - 1]),
         ("max", 2 * mx + 100, [mx]),                        # cut at max by the rule, then skipped (= next start)
         ("eof-last-byte", f + 700, [f + 699])]
    gaps = [min_eff, min_eff + 1, mx - 1, mx, (min_eff + mx) // 2]
    pos, p = [], f
    for g in gaps * 2:                                       # every candidate a cut
        pos.append(p)
        p += g
    S.append(("spaced-cuts", p + 77, pos))
    # a mix of skipped and cut candidates (two patterns closer than 65 bytes would share a window: no gap of 64 at avg 256)
    gaps = [max(min_eff - 1, 65), mx + 1, min_eff, 2 * min_eff - 1, mx - 1]
    pos, p = [], f
    for g in gaps * 2:
        pos.append(p)
        p += g
    S.append(("spaced-mixed", p + 1, pos))
    return S


def _build(streams, avg):
    pat = _pattern(avg)
    return [sr.plant(n, pos, pat) for _, n, pos in streams], [sr.expected_candidates(pos) for _, _, pos in streams]


def _pack(arrs, lead):
    off, pos = [], lead
    for a in arrs:
        off.append(pos)
        pos += (len(a) + 127) // 128 * 128 + 128
    buf = np.zeros(pos + 64, dtype=np.uint8)
    for a, o in zip(arrs, off):
        buf[o:o + len(a)] = a
    return buf, np.array(off, dtype=np.uint64), np.array([len(a) for a in arrs], dtype=np.uint64)


# ---- expectations -----------------------------------------------------------------------------------------------------
def _sha(chunk, memo):
    """SHA-256 of a chunk; all-zero chunks of one length share one digest, hashed once."""
    if not chunk.any():
        if len(chunk) not in memo:
            memo[len(chunk)] = hashlib.sha256(chunk).digest()
        return memo[len(chunk)]
    return hashlib.sha256(chunk).digest()


def _expect(arrs, cands, cfg, forced=None):
    """(ends, stream_first, chunk records) that K2 and K3 must produce for these streams."""
    ends, first, rows, memo = [], [0], [], {}
    for s, (a, c) in enumerate(zip(arrs, cands)):
        e = sr.resolve(c, len(a), cfg, forced=(forced or {}).get(s, ()))
        start = 0
        for x in e:
            rows.append((s, x, _sha(a[start:x], memo)))
            start = x
        ends += e
        first.append(len(ends))
    rec = np.zeros(len(rows), dtype=pg.CHUNK_DTYPE)
    for i, (s, x, d) in enumerate(rows):
        rec[i]["stream"], rec[i]["end_off"], rec[i]["digest"] = s, x, np.frombuffer(d, dtype=np.uint8)
    return ends, first, rec


def _first_diff(got_ends, got_first, want_ends, want_first, streams):
    """The first stream whose cut list differs, for the failure message."""
    for s in range(len(streams)):
        g = list(got_ends[int(got_first[s]):int(got_first[s + 1])]) if s + 1 < len(got_first) else None
        w = want_ends[want_first[s]:want_first[s + 1]]
        if g != w:
            cls, n, pos = streams[s]
            return f"stream {s} ({cls}, len {n}, planted {pos[:6]}): got {g[:8] if g else g}, want {w[:8]}"
    return "stream_first differs"


def _check_records(rec, want, streams, what):
    if rec.tobytes() == want.tobytes():
        return
    for i in range(min(len(rec), len(want))):
        if rec[i].tobytes() != want[i].tobytes():
            s = int(want[i]["stream"])
            raise AssertionError(f"{what}: record {i} differs (stream {s}, {streams[s][0]}): got stream "
                                 f"{int(rec[i]['stream'])} end {int(rec[i]['end_off'])} flags {int(rec[i]['flags'])}, "
                                 f"want end {int(want[i]['end_off'])}")
    raise AssertionError(f"{what}: {len(rec)} records, want {len(want)}")


def _run_all_checks(torch, e, cfg, arrs, cands, streams, lead, what):
    want_e, want_f, want_rec = _expect(arrs, cands, cfg)
    buf, off, ln = _pack(arrs, lead)
    dev = torch.from_numpy(buf).cuda()
    ends, first = e.scan_batch(cfg, dev, off, ln)
    assert ends.tolist() == want_e and first.tolist() == want_f, (what, _first_diff(ends, first, want_e, want_f, streams))
    rec, t = e.submit(cfg, dev, off, ln).wait()
    n_cand = sum(len(c) for c in cands)
    assert t["candidates"] == n_cand, (what, "K1 candidates", t["candidates"], n_cand)
    _check_records(rec, want_rec, streams, what)


# ---- tests ------------------------------------------------------------------------------------------------------------
def test_the_matrix_covers_every_edge_class():
    """Every listed edge class is planted; every planted position of a class is a reference candidate (or 62)."""
    streams = _kernel_edge_streams()
    classes = {c for c, _, _ in streams}
    for k, want in KERNEL_EDGE_CLASSES.items():
        assert want <= classes, (k, want - classes)
    for cls, n, pos in streams:
        assert all(p < n for p in pos) and (cls == "first-window" or all(p >= 63 for p in pos)), (cls, pos)
    assert {v for c, n, _ in streams if c.startswith("partial-tile") for v in [n % TILE]} == {1, 271, 272, 273, 8703}
    rules = {c for c, _, _ in _rule_edge_streams(4096)}
    assert {"first_ok-1", "first_ok", "max-1", "max", "eof-last-byte", "spaced-cuts"} <= rules


@pytest.mark.parametrize("avg", AVGS)
@pytest.mark.parametrize("kernel", KERNELS)
def test_kernel_edges(torch, engines, kernel, avg):
    streams = _kernel_edge_streams()
    arrs, cands = _build(streams, avg)
    cfg = _cfg(avg)
    with _kernel(engines, kernel) as e:
        for layout, lead in LAYOUTS.items():
            _run_all_checks(torch, e, cfg, arrs, cands, streams, lead, (kernel, avg, layout))


@pytest.mark.parametrize("avg", AVGS)
@pytest.mark.parametrize("kernel", KERNELS)
def test_min_max_rule_edges(torch, engines, kernel, avg):
    streams = _rule_edge_streams(avg)
    arrs, cands = _build(streams, avg)
    cfg = _cfg(avg)
    layouts = LAYOUTS if avg < 1 << 22 else {"aligned128": 0}     # 16 MiB chunks: one layout keeps the SHA-256 time small
    with _kernel(engines, kernel) as e:
        for layout, lead in layouts.items():
            _run_all_checks(torch, e, cfg, arrs, cands, streams, lead, (kernel, avg, layout))


@pytest.mark.parametrize("avg", [512, 4096, 1 << 16])
@pytest.mark.parametrize("kernel", KERNELS)
def test_forced_boundaries_on_rule_edges(torch, engines, kernel, avg):
    """A suggested boundary whose key equals a hash candidate, one at first_ok - 1 (skipped), one at first_ok, and
    one in a chunk that a candidate cuts first."""
    cfg = _cfg(avg)
    min_eff, mx = max(int(cfg.min), 65), int(cfg.max)
    f = min_eff - 1
    streams = [("forced-equals-candidate", mx + 500, [f + 10]),
               ("forced-at-first_ok-1", mx + 500, []),
               ("forced-at-first_ok", mx + 500, []),
               ("forced-after-candidate", mx + 500, [f + 10])]
    forced = {0: [f + 11], 1: [f], 2: [f + 1], 3: [f + 200]}
    arrs = [sr.plant(n, pos, _pattern(avg)) if pos else np.zeros(n, dtype=np.uint8) for _, n, pos in streams]
    cands = [sr.expected_candidates(pos) for _, _, pos in streams]
    want_e, _, want_rec = _expect(arrs, cands, cfg, forced)
    fs = np.array([s for s in sorted(forced) for _ in forced[s]], dtype=np.uint32)
    fo = np.array([b for s in sorted(forced) for b in forced[s]], dtype=np.uint64)
    buf, off, ln = _pack(arrs, 0)
    with _kernel(engines, kernel) as e:
        rec = e.chunk_digest_batch(cfg, torch.from_numpy(buf).cuda(), off, ln, forced=(fs, fo))
    assert rec["end_off"].tolist() == want_e
    _check_records(rec, want_rec, streams, (kernel, avg, "forced"))
    for s, a in enumerate(arrs):                              # the oracle's own forced-boundary chunker agrees
        assert oracle.chunk_digest_forced(oracle.config(avg), a, forced[s])["end_off"].tolist() == \
            sr.resolve(cands[s], len(a), cfg, forced=forced[s])


@pytest.mark.parametrize("kernel", KERNELS)
def test_host_batch_staged_in_groups(torch, kernel):
    """Host input staged in several groups of 256 KiB: the same records as from device memory."""
    env = {"PBSGPU_STAGE_BYTES": str(1 << 18)}
    if kernel == "lanes":
        env["PBSGPU_SCAN_LANES"] = "1"
    e = _engine_with_env(env)
    try:
        e.set_kernel_variant(1 if kernel == "simple" else 0)
        for avg in (256, 4096):
            streams = _kernel_edge_streams() + _rule_edge_streams(avg)
            arrs, cands = _build(streams, avg)
            cfg = _cfg(avg)
            _, _, want = _expect(arrs, cands, cfg)
            buf, off, ln = _pack(arrs, 0)
            _check_records(e.chunk_digest_batch(cfg, buf, off, ln), want, streams, (kernel, avg, "staged"))
    finally:
        e.close()


@pytest.mark.parametrize("kernel", KERNELS)
def test_stream_writer_window_ends_at_planted_candidates(kernel):
    """The stream writer scans each full window with eof = 0 and carries the undecided tail; the first window's last
    byte falls at P - 1, P and P + 63 of a planted candidate P, and writes are split around P."""
    W, avg = 100_000, 4096                                    # not a multiple of max: the candidates are cuts
    env = {"PBSGPU_STREAM_WINDOW": str(W)}
    if kernel == "lanes":
        env["PBSGPU_SCAN_LANES"] = "1"
    e = _engine_with_env(env)
    try:
        e.set_kernel_variant(1 if kernel == "simple" else 0)
        cfg = _cfg(avg)
        assert W >= cfg.max
        for P in (W, W - 1, W - 64):                         # window's last byte W - 1 = P - 1, P, P + 63
            n = 3 * W + 1234
            pos = [P, 2 * W + 5000, n - 1]
            a = sr.plant(n, pos, _pattern(avg))
            _, _, want = _expect([a], [sr.expected_candidates(pos)], cfg)
            st = e.stream(cfg)
            at = 0
            for size in (P - 1, 1, 1, 63, 10 ** 9):
                st.write(a[at:at + size])
                at = min(n, at + size)
            rec = st.finish()
            st.close()
            _check_records(rec, want, [("stream-window", n, pos)], (kernel, "stream", P - W))
    finally:
        e.close()


def test_avg_2_29_chunk_of_exactly_max(torch, engines):
    """Average 2^29 (a purpose-made table: the default one has no suitable pattern at mask 2^30 - 1): one stream of
    2^31 + 4097 bytes whose first chunk is max = 2^31 bytes long, the ChunkRef.len limit, cut by a candidate on its
    last byte and, in a second pass, by the max rule alone.  Cut lists only: a 2 GiB chunk is one serial SHA-256 chain."""
    avg, n = 1 << 29, (1 << 31) + 4097
    free, _ = torch.cuda.mem_get_info()
    if free < n + (4 << 30):
        pytest.skip(f"needs about {(n >> 30) + 4} GiB of free device memory, {free >> 30} GiB free")
    cfg, pat = _cfg(avg), _pattern(avg)
    f = max(int(cfg.min), 65) - 1
    dev = torch.zeros(n, dtype=torch.uint8, device="cuda")
    pb = torch.tensor(list(pat.bytes), dtype=torch.uint8, device="cuda")
    for pos in ([f - 1, (1 << 31) - 1, (1 << 31) + 100, n - 1], [f - 1, (1 << 31) + 100, n - 1]):
        dev.zero_()
        for o in sr.offsets_for(pos, pat):
            dev[o:o + 3] = pb
        got = lambda lo, hi: dev[lo:hi].cpu().numpy()
        want = sr.resolve(sr.check_planted(got, n, pos, pat), n, cfg)
        assert want == [1 << 31, n]
        for k in KERNELS:
            with _kernel(engines, k) as e:
                ends, first = e.scan_batch(cfg, dev, [0], [n])
            assert ends.tolist() == want and first.tolist() == [0, 2], (k, pos, ends.tolist())
    del dev
    torch.cuda.empty_cache()


def test_one_stream_past_2_32_bytes(torch, engines):
    """One device stream of 2^32 + 2^22 + 5 bytes at average 4 MiB: candidates at 2^32 - 1, 2^32, 2^32 + 271 and at the
    first tile and super-tile edges past 2^32 must come back at their 40-bit positions (a position truncated to 32
    bits would land before the first cut and vanish).  An early candidate shifts the max-rule cuts off the 2^24 grid
    so that each of those candidates is a cut.  Then the digests, the stream's XXH3-64 and fixed 4 MiB records."""
    avg, n = 1 << 22, (1 << 32) + (1 << 22) + 5
    free, _ = torch.cuda.mem_get_info()
    if free < n + (4 << 30):
        pytest.skip(f"needs about {(n >> 30) + 4} GiB of free device memory, {free >> 30} GiB free")
    cfg, pat = _cfg(avg), _pattern(avg)
    G = 1 << 32
    phase = (1 << 23) + 4097
    tile_past = -(-G // TILE) * TILE
    dev = torch.zeros(n, dtype=torch.uint8, device="cuda")
    pb = torch.tensor(list(pat.bytes), dtype=torch.uint8, device="cuda")
    got = lambda lo, hi: dev[lo:hi].cpu().numpy()
    planted = []
    for P in (G - 1, G, G + 271, tile_past, G + SUPER, n - 1):
        pos = [phase, P]
        planted = pos
        dev.zero_()
        for o in sr.offsets_for(pos, pat):
            dev[o:o + 3] = pb
        want = sr.resolve(sr.check_planted(got, n, pos, pat), n, cfg)
        assert P + 1 in want or P == n - 1, (P, want[-4:])
        for k in KERNELS:
            with _kernel(engines, k) as e:
                ends, first = e.scan_batch(cfg, dev, [0], [n])
            assert ends.tolist() == want and first.tolist() == [0, len(want)], (k, P, ends.tolist()[-4:], want[-4:])
    e = engines["tuned"][0]
    host = dev.cpu().numpy()
    _, _, want_rec = _expect([host], [sr.expected_candidates(planted)], cfg)
    rec, h = e.chunk_digest_batch_xxh3(cfg, dev, [0], [n])
    _check_records(rec, want_rec, [("past-2^32", n, planted)], "past 2^32 digests")
    assert int(h[0]) == oracle.xxh3_64(host)
    fixed = e.chunk_digest_batch(None, dev, [0], [n], fixed_size=4 << 20)          # the .fidx chunking
    ends = [min(n, k) for k in range(4 << 20, n + (4 << 20), 4 << 20)]
    assert fixed["end_off"].tolist() == ends
    memo, start = {}, 0
    for r, x in zip(fixed, ends):
        assert bytes(r["digest"]) == _sha(host[start:x], memo), x
        start = x
    del dev, host
    torch.cuda.empty_cache()
