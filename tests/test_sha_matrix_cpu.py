"""The K3 matrix covers what ships: every mode arm of csrc/sha256.cu's launch switches is in sha_matrix.MODES, every
K3 knob capi.cu reads at open is set by sha_matrix.PATHS or KERNELS, and the matrix's inputs reach the edges they are
meant to.  A new instantiation or knob that nobody adds to the matrix fails here, on any machine."""
import re
from pathlib import Path

import numpy as np

import sha_matrix as M

CSRC = Path(__file__).resolve().parent.parent / "pbs_plus_b200" / "csrc"


def function_body(src: str, signature: str) -> str:
    """The text of the function whose definition starts with `signature`, up to its closing brace at column 0."""
    i = src.index(signature)
    return src[i: src.index("\n}\n", i)]


def switches(body: str) -> list[str]:
    """The switch statements of a function body, each up to the next switch (or the end of the body)."""
    parts = re.split(r"\bswitch\s*\(tune\.mode\)", body)
    assert len(parts) >= 2, "no switch on tune.mode"
    return parts[1:]


def cases(sw: str) -> set[int]:
    return {int(m) for m in re.findall(r"\bcase\s+(\d+)\s*:", sw)}


def test_every_mode_arm_is_in_the_matrix():
    src = (CSRC / "sha256.cu").read_text()
    tuned = switches(function_body(src, "cudaError_t launch_sha_tuned("))
    split = switches(function_body(src, "cudaError_t launch_sha_split("))
    assert len(tuned) == 2 and len(split) == 1
    keyed, plain = tuned
    # the keyed and the plain switch have the same arms, and arm N launches the mode-N kernel of its kind
    assert cases(keyed) == cases(plain)
    for sw, kind in ((keyed, "true"), (plain, "false")):
        for n, m, k in re.findall(r"\bcase\s+(\d+)\s*:\s*k_sha_tuned<(\d+),\s*(\w+)>", sw):
            assert (n, k) == (m, kind), (n, m, k)
        assert len(re.findall(r"\bcase\s+\d+\s*:\s*k_sha_tuned<", sw)) == len(cases(sw))
    # the throughput default arm runs mode 2's kernel; the split default runs every mode >= 10 without an arm: 11
    tuned_default = {int(m) for m in re.findall(r"default\s*:\s*k_sha_tuned<(\d+),", keyed + plain)}
    assert tuned_default == {2} and 2 not in cases(keyed)
    assert "default:" in split[0] and 11 not in cases(split[0]) and min(cases(split[0])) >= 10
    shipped = cases(keyed) | tuned_default | cases(split[0]) | {11}
    assert shipped == set(M.MODES), sorted(shipped ^ set(M.MODES))
    assert len(M.MODES) == len(set(M.MODES))
    # the simple cross-check kernel has its plain and keyed forms, selected by PBSGPU_VARIANT=1
    assert "k_sha_simple_keyed" in src and M.KERNELS["simple"] == {"PBSGPU_VARIANT": "1"}
    assert {k: v for k, v in M.KERNELS.items() if k != "simple"} == {f"mode{m}": {"PBSGPU_SHA_MODE": str(m)} for m in M.MODES}


def test_every_k3_knob_is_in_the_matrix():
    src = (CSRC / "capi.cu").read_text()
    knobs = set(re.findall(r"ctx->tune\.\w+\s*=[^;]*env_int\(\"(PBSGPU_\w+)\"", src))
    assert {"PBSGPU_SHA_MODE", "PBSGPU_SHA_HYBRID", "PBSGPU_HYBRID_SERIAL"} <= knobs, knobs
    assert re.search(r"env_int\(\"PBSGPU_VARIANT\"", src)
    knobs.add("PBSGPU_VARIANT")
    set_by_paths = {k for env in M.PATHS.values() for k in env}
    set_by_kernels = {k for env in M.KERNELS.values() for k in env}
    assert knobs - {"PBSGPU_SHA_MODE"} <= set_by_paths, sorted(knobs - set_by_paths)
    assert knobs <= set_by_paths | set_by_kernels


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
    # the mid path: a head of chunks over 2 x avg and a non-empty mid class behind it
    env = M.PATHS["mid"]
    head = M.split_point(lens, int(env["PBSGPU_HYBRID_THR_X10"]))
    mid = M.split_point(lens, int(env["PBSGPU_BULK_MID_X10"]))
    assert 0 < head < mid < n
    assert M.fixed_cuts(parts, 1 << 18)[-1] == (len(parts) - 1, len(parts[-1]))
    assert np.all(np.array([e for _, e in M.fixed_cuts(parts, 1 << 18)]) > 0)
