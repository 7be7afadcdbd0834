"""The matrix that pins K3 (csrc/sha256.cu): every kernel, every launch path, the inputs that put each one at its
edges, and the hashlib reference.  Importing it needs no GPU; test_gpu_sha_matrix.py runs the matrix and
test_sha_matrix_cpu.py fails when sha256.cu or capi.cu gains a kernel instantiation or a knob that is not listed here.

- KERNELS: the kernels of the blocking byte-range calls: the throughput kernel (k_sha_tuned, the default) and the
  simple cross-check kernel (PBSGPU_VARIANT=1).
- PATHS: the K3 launch paths of the batch job, as the environment a context is opened with.  The latency kernel
  (k_sha_split) runs on the hybrid ones; "split_every_chunk" (without the SM partition) and
  "split_every_chunk_partitioned" (on the long-chunk partition) give it every chunk of a job.
- The reference is hashlib: SHA-256(chunk), and SHA-256(chunk || id_key) for encrypt mode's keyed digests, with
  id_key from crypt_ref (PBKDF2 in hashlib).  Nothing from the library computes an expected value.
"""
from __future__ import annotations

import hashlib

import numpy as np

import crypt_ref

KERNELS = {"tuned": {}, "simple": {"PBSGPU_VARIANT": "1"}}

AVG = 1 << 16                     # the streams' chunker: min 16 KiB, max 256 KiB = 4 x AVG
MAX_OVER_AVG_X10 = 40
# the split point, for the job paths below: (first index with len <= thr rounded up to 32) capped at the head limit and n
SPLIT_AT = {"split_none": MAX_OVER_AVG_X10, "split_32k": MAX_OVER_AVG_X10 - 1, "split_all": 1}

PATHS = {
    "throughput": {"PBSGPU_SHA_HYBRID": "0"},
    "hybrid_nopart": {"PBSGPU_SHA_HYBRID": "2", "PBSGPU_PARTITION_SMS": "0"},
    "partitioned": {},
    "spread0": {"PBSGPU_SPLIT_SPREAD_KB": "0"},
    "spread85": {"PBSGPU_SPLIT_SPREAD_KB": "85"},
    # 1 x 24 chunks rounded down to whole CTAs of 32: the split kernel launches with an empty head
    "head_per_sm1": {"PBSGPU_SHA_HYBRID": "2", "PBSGPU_PARTITION_SMS": "0", "PBSGPU_HYBRID_HEAD_PER_SM": "1"},
    # threshold 0 and a head limit of 64 x 24 chunks (24: the default partition's SMs, and the count assumed without
    # one): every chunk of a job with up to 1536 of them takes the latency kernel
    "split_every_chunk": {"PBSGPU_SHA_HYBRID": "2", "PBSGPU_PARTITION_SMS": "0", "PBSGPU_HYBRID_THR_X10": "0",
                          "PBSGPU_HYBRID_HEAD_PER_SM": "64"},
    "split_every_chunk_partitioned": {"PBSGPU_HYBRID_THR_X10": "0", "PBSGPU_HYBRID_HEAD_PER_SM": "64"},
    "variant1": {"PBSGPU_VARIANT": "1"},
    **{name: {"PBSGPU_HYBRID_THR_X10": str(thr)} for name, thr in SPLIT_AT.items()},
}

KEY = bytes(range(53, 85))
IDENT = crypt_ref.id_key(KEY)


def digest(data, keyed: bool = False) -> bytes:
    """The reference: SHA-256(data), or SHA-256(data || id_key(KEY)) when keyed."""
    return hashlib.sha256(bytes(data) + (IDENT if keyed else b"")).digest()


def layout(lens, residues, shift: int = 0):
    """(buffer, offsets, lengths) of random ranges of `lens`, range i starting at residues[i] mod 16, one or more
    bytes apart so that no two ranges share a 16-byte vector edge by accident."""
    offs, pos = [], shift
    for n, r in zip(lens, residues):
        pos += 1 + (r - pos - 1) % 16
        offs.append(pos)
        pos += n
    buf = np.random.default_rng(len(lens) + shift).integers(0, 256, size=pos + 64, dtype=np.uint8)
    return buf, np.array(offs, np.uint64), np.array(lens, np.uint64)


def edge_lens() -> tuple[list[int], list[int]]:
    """(lengths, start residues mod 16): 0..300 twice, each length mod 64 at several start residues, 64k + d around
    the padding edges for k in {5, 16, 63, 64}, then 64k + r for every r in 0..63 and k in {4, 17, 1000}.  The keyed
    suffix moves the one-or-two final block boundary from len % 64 = 56 to 24, and for residues 33..63 the suffix
    itself crosses a block edge."""
    lens, res = [], []
    for half in (0, 8):
        for n in range(301):
            lens.append(n)
            res.append((n + 7 * (n // 64) + half) % 16)
    for k in (5, 16, 63, 64):
        for d in (-9, -8, -1, 0, 1, 55, 56):
            lens.append(64 * k + d)
            res.append((k + 3 * d) % 16)
    for ki, k in enumerate((4, 17, 1000)):
        for r in range(64):
            lens.append(64 * k + r)
            res.append((3 * r + 5 * ki) % 16)
    return lens, res


def edges():
    return layout(*edge_lens())


# The edge set as streams of one chunk each: at this average the minimum chunk (avg / 4) is longer than any edge
# range, so every stream ends in its EOF chunk, which may have any length.
EDGE_AVG = 1 << 18
# Messages of 512 MiB - 1, 512 MiB and 512 MiB + 1 as all-zero streams: a zero background has no boundary candidate
# (scan_ref), so each is one chunk, and at this average (maximum 2 GiB) the job takes them whole.
LONG_AVG = 1 << 29
LONG_ZERO = [(1 << 29) - 1, 1 << 29, (1 << 29) + 1]


def long_lens() -> list[int]:
    """A few multi-MiB ranges for the split kernels' many-block chains, at both keyed finish forms."""
    return [(3 << 20) + 5, (4 << 20) + 23, (4 << 20) + 24, (5 << 20) + 63, 6 << 20, 8 << 20]


def edges_and_long():
    """The edge set followed by the long set in one buffer: short and long lanes share the warps of one launch."""
    lens, res = edge_lens()
    ll = long_lens()
    return layout(lens + ll, res + [(5 * i + 3) % 16 for i in range(len(ll))], shift=3)


# ---- the batch job's streams ----------------------------------------------------------------------------------
def stream_parts() -> list[np.ndarray]:
    """Random streams with zero runs (the chunker cuts them at the maximum, 4 x AVG), a short stream and an empty
    one: about ten maximum-length chunks among a few hundred, so that the SPLIT_AT thresholds put the split point at
    0, at a multiple of 32 short of n and at n (n itself not a multiple of 32) (test_sha_matrix_cpu checks each)."""
    rng = np.random.default_rng(31)
    parts = []
    for i in range(6):
        a = rng.integers(0, 256, size=2_600_000 + 4099 * i, dtype=np.uint8)
        if i % 2 == 0:
            a[300_000 + 1000 * i: 300_000 + 1000 * i + 1_000_000] = 0
        parts.append(a)
    parts.append(np.zeros(0, np.uint8))
    parts.append(rng.integers(0, 256, size=777, dtype=np.uint8))
    return parts


def pack_streams(parts):
    """((buffer, offsets, lengths), parts): the streams in one buffer, stream i starting at residue 3 * i mod 16."""
    buf, off, ln = layout([len(p) for p in parts], [(3 * i) % 16 for i in range(len(parts))])
    for p, o in zip(parts, off):
        buf[int(o): int(o) + len(p)] = p
    return (buf, off, ln), parts


def records(cuts: np.ndarray, parts, keyed: bool) -> np.ndarray:
    """`cuts` (records with stream and end_off) with every digest recomputed by hashlib from the chunk bytes."""
    out = cuts.copy()
    prev = {}
    for r in out:
        s, e = int(r["stream"]), int(r["end_off"])
        b = prev.get(s, 0)
        r["digest"] = np.frombuffer(digest(parts[s][b:e], keyed), np.uint8)
        prev[s] = e
    return out


def chunk_lens(rec: np.ndarray) -> np.ndarray:
    ends = rec["end_off"].astype(np.int64)
    st = rec["stream"].astype(np.int64)
    first = np.r_[True, st[1:] != st[:-1]]
    return ends - np.where(first, 0, np.r_[0, ends[:-1]])


def split_point(lens: np.ndarray, thr_x10: int, max_head: int = 768) -> int:
    """k_split_point restated: the count of chunks longer than thr_x10 / 10 x AVG, rounded up to 32, capped at
    max_head (rounded down to 32) and at n."""
    n = len(lens)
    h = (int((lens > AVG * thr_x10 // 10).sum()) + 31) & ~31
    if h > max_head:
        h = max_head & ~31
    return min(h, n)


def fixed_cuts(parts, size: int) -> list[tuple[int, int]]:
    """(stream, end) of fixed-size chunks: every `size` bytes, the last one short."""
    return [(s, min(e, len(p))) for s, p in enumerate(parts) for e in range(size, len(p) + size, size)]
