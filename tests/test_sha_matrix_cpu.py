"""The K3 matrix covers what ships: csrc/sha256.cu has one throughput and one latency kernel, each plain and keyed,
every K3 knob capi.cu reads at open is set by sha_matrix.PATHS or KERNELS, and the matrix's inputs reach the edges they
are meant to.  A new instantiation or knob that nobody adds to the matrix fails here, on any machine."""
import re
from pathlib import Path

import numpy as np

import sha_matrix as M

CSRC = Path(__file__).resolve().parent.parent / "pbs_plus_b200" / "csrc"
# every variable capi.cu reads: a knob added or brought back fails here until it is listed (and, for K3, in the matrix)
CAPI_ENV = {"PBSGPU_ARENA_FRAC_X16", "PBSGPU_ARENA_MB", "PBSGPU_DEBUG", "PBSGPU_HYBRID_HEAD_PER_SM", "PBSGPU_HYBRID_THR_X10",
            "PBSGPU_KEEP_ENV", "PBSGPU_PARTITION_SMS", "PBSGPU_SCAN_LANES", "PBSGPU_SCAN_SMS", "PBSGPU_SHA_HYBRID",
            "PBSGPU_SLOTS", "PBSGPU_SPLIT_SPREAD_KB", "PBSGPU_STAGE_BYTES", "PBSGPU_STREAM_NBUF", "PBSGPU_STREAM_WINDOW",
            "PBSGPU_VARIANT", "PBSGPU_XXH3_CAP_BLOCKS"}


def test_one_kernel_instantiation_per_keyed_value():
    src = (CSRC / "sha256.cu").read_text()
    # the kernels take KEYED as their only template parameter, and every use names one of its two values
    for k in ("k_sha_tuned", "k_sha_split"):
        assert len(re.findall(rf"\b{k}\(", src)) == 1, k
        assert re.search(rf"template <bool KEYED>\n__global__ void __launch_bounds__\(\d+\) {k}\(", src), k
        uses = re.findall(rf"\b{k}<([^>]*)>", src)
        assert uses and set(uses) == {"true", "false"}, (k, uses)
    assert "k_sha_simple_keyed" in src and M.KERNELS == {"tuned": {}, "simple": {"PBSGPU_VARIANT": "1"}}


def test_capi_reads_only_listed_knobs_and_the_matrix_sets_every_k3_knob():
    src = (CSRC / "capi.cu").read_text()
    knobs = set(re.findall(r"ctx->tune\.\w+\s*=[^;]*env_int\(\"(PBSGPU_\w+)\"", src))
    assert {"PBSGPU_SHA_HYBRID", "PBSGPU_HYBRID_THR_X10", "PBSGPU_SPLIT_SPREAD_KB", "PBSGPU_HYBRID_HEAD_PER_SM"} <= knobs, knobs
    assert re.search(r"env_int\(\"PBSGPU_VARIANT\"", src)
    knobs.add("PBSGPU_VARIANT")
    set_by_paths = {k for env in M.PATHS.values() for k in env}
    assert knobs <= set_by_paths, sorted(knobs - set_by_paths)
    assert set(re.findall(r"\"(PBSGPU_\w+)\"", src)) == CAPI_ENV


def test_edge_inputs_reach_every_padding_form_and_alignment():
    lens, res = M.edge_lens()
    buf, off, ln = M.edges()
    assert ln.tolist() == lens and [int(o) % 16 for o in off] == res
    assert set(res) == set(range(16))
    for k in (0, 1, 2, 3, 4, 17, 1000):
        assert {n % 64 for n in lens if n // 64 == k} == set(range(64)), k
    for r in range(64):   # each length residue at several start residues
        assert len({s for n, s in zip(lens, res) if n % 64 == r}) >= 4, r
    assert all(o + n <= len(buf) for o, n in zip(off.tolist(), lens))
    buf, off, ln = M.edges_and_long()
    assert ln.tolist()[-len(M.long_lens()):] == M.long_lens()
    assert {n % 64 for n in M.long_lens()} >= {23, 24, 63}   # keyed: one final block, two, suffix across the edge


def test_edge_and_zero_streams_are_one_chunk_each_and_all_in_the_latency_kernels_head():
    import oracle
    import scan_ref
    buf, off, ln = M.edges()
    lens = ln.tolist()
    assert max(lens) < M.EDGE_AVG // 4   # below the minimum chunk: no cut
    cuts = oracle.chunk_digest_streams(oracle.config(M.EDGE_AVG), [buf[int(o): int(o) + n] for o, n in zip(off, lens)])
    assert cuts["end_off"].tolist() == [n for n in lens if n]
    env = M.PATHS["split_every_chunk"]
    assert M.PATHS["split_every_chunk_partitioned"].items() <= env.items()
    max_head = int(env["PBSGPU_HYBRID_HEAD_PER_SM"]) * 24
    assert M.split_point(M.chunk_lens(cuts), int(env["PBSGPU_HYBRID_THR_X10"]), max_head) == len(cuts)
    assert M.split_point(np.array(M.LONG_ZERO), 0, max_head) == 3
    # plain bit lengths below, at and above 2^32; keyed above; all within the maximum chunk
    assert [8 * n >= 1 << 32 for n in M.LONG_ZERO] == [False, True, True] and max(M.LONG_ZERO) <= 4 * M.LONG_AVG
    assert len(scan_ref.candidates(oracle.default_table(), oracle.config(M.LONG_AVG).mask, np.zeros(1 << 20, np.uint8))) == 0


def test_stream_inputs_put_the_split_point_at_its_edges():
    import oracle
    (buf, off, ln), parts = M.pack_streams(M.stream_parts())
    for p, o in zip(parts, off):
        assert (buf[int(o): int(o) + len(p)] == p).all()
    lens = M.chunk_lens(oracle.chunk_digest_streams(oracle.config(M.AVG), parts))
    n = len(lens)
    assert n % 32 and n <= 768
    assert (lens == 4 * M.AVG).sum() >= 8   # zero runs cut at the maximum
    at = {name: M.split_point(lens, thr) for name, thr in M.SPLIT_AT.items()}
    assert at["split_none"] == 0 and at["split_all"] == n
    assert at["split_32k"] % 32 == 0 and 0 < at["split_32k"] < n
    # the default threshold has a head; the head limit of 1 x 24 chunks empties it
    assert M.split_point(lens, 25) > 0 and M.split_point(lens, 25, max_head=24) == 0
    assert M.fixed_cuts(parts, 1 << 18)[-1] == (len(parts) - 1, len(parts[-1]))
    assert np.all(np.array([e for _, e in M.fixed_cuts(parts, 1 << 18)]) > 0)
