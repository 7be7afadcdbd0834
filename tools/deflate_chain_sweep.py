"""The sweep behind the constants of the Deflate chain parse (tests/deflate_chain_ref.py, DESIGN.md K16d): stream size /
input for every (MINMATCH, TOO_FAR, DEPTH, LAZY, MARGIN) row, the greedy parse of pbsgpu_deflate_batch, and zlib
levels 1, 4 and 6 per 128 KiB segment, on the text, binary, repeated and half-zero corpora.  CPU only.

Sizes come from each segment's symbol histograms with tests/deflate_ref.py's cost rules (the smallest of the stored,
fixed and dynamic forms with the segment's end), which equal len(deflate_chain_ref.deflate(...)); --check confirms that
on the first MiB of each corpus.

    python tools/deflate_chain_sweep.py [--sizes 1,8] [--jobs 8] [--check]"""
from __future__ import annotations

import argparse
import itertools
import os
import sys
import zlib
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, ".."), os.path.join(HERE, "..", "tests")]

import deflate_chain_ref as ch  # noqa: E402
import deflate_ref as dr  # noqa: E402
import zstd_chain_ref as zch  # noqa: E402
import zstd_huf_ref as hufref  # noqa: E402
import zstd_ldm_ref as ldm  # noqa: E402
import zstd_lz_ref as lzref  # noqa: E402

DEPTHS, LAZIES, MARGINS = (4, 8, 16, 32), (0, 1, 2), (0, 4, 8)
MATCH_RULES = ((3, 0), (3, 4096), (4, 0))   # (MINMATCH, TOO_FAR)
LEN_CODE = np.array([0, 0, 0] + [dr.len_code(L) - 257 for L in range(3, 259)])
LEN_EXTRA = np.array(dr.LEN_BITS)
DIST_CODE = np.array([0] + [dr.dist_code(d) for d in range(1, 32769)])
DIST_EXTRA = np.array(dr.DIST_BITS)
FIXED_LIT, FIXED_DIST = np.array(dr.FIXED_LIT), np.array(dr.FIXED_DIST)


def corpus(name: str, n: int) -> bytes:
    if name == "text":
        return bytes(lzref.text_corpus(n, 1))
    if name == "binary":
        return bytes(hufref.binary_corpus(n, 2))
    if name == "repeated":
        return bytes(ldm.repeated_image(hufref.binary_corpus(256 << 10, 3), n // (256 << 10), n // 512, 4))
    return bytes(zch.half_zero(n, 5))


def segment_bytes(seg: np.ndarray, seqs, final: bool) -> int:
    """deflate_ref.encode_segment's output size for the segment's matches [(pos in segment, L, offset)]."""
    S = len(seg)
    cover = np.zeros(S + 1, np.int64)
    lit_cnt, dist_cnt = np.zeros(286, np.int64), np.zeros(30, np.int64)
    if seqs:
        m, L, o = (np.array(x, np.int64) for x in zip(*seqs))
        np.add.at(cover, m, 1)
        np.add.at(cover, m + L, -1)
        np.add.at(lit_cnt, 257 + LEN_CODE[L], 1)
        np.add.at(dist_cnt, DIST_CODE[o], 1)
        extra = int(LEN_EXTRA[LEN_CODE[L]].sum() + DIST_EXTRA[DIST_CODE[o]].sum())
    else:
        extra = 0
    lit_cnt[:256] += np.bincount(seg[np.cumsum(cover[:S]) == 0], minlength=256)
    lit_cnt[256] += 1
    nst = (S + dr.STORED_MAX - 1) // dr.STORED_MAX
    stored = 40 * nst + 8 * S
    fixed = 3 + int((lit_cnt * FIXED_LIT[:286]).sum() + (dist_cnt * FIXED_DIST).sum()) + extra
    lit_len = dr.huffman_lengths(lit_cnt.tolist(), dr.LIT_MAXBITS)
    dist_len = dr.huffman_lengths(dist_cnt.tolist(), dr.LIT_MAXBITS)
    hlit = max(257, max(s for s in range(286) if lit_len[s]) + 1)
    if any(dist_len):
        hdist = max(s for s in range(30) if dist_len[s]) + 1
    else:
        dist_len[0], hdist = 1, 1
    runs = dr.cl_runs(lit_len[:hlit] + dist_len[:hdist])
    cl_cnt = [0] * 19
    for s, _, _ in runs:
        cl_cnt[s] += 1
    cl_len = dr.huffman_lengths(cl_cnt, dr.CL_MAXBITS)
    hclen = 19
    while hclen > 4 and cl_len[dr.CL_ORDER[hclen - 1]] == 0:
        hclen -= 1
    hdr = 3 + 14 + 3 * hclen + sum(cl_len[s] + nb for s, _, nb in runs)
    dyn = hdr + int((lit_cnt * np.array(lit_len)).sum() + (dist_cnt * np.array(dist_len)).sum()) + extra

    def total(b):
        return (b + 7) // 8 * 8 if final else (b + 3 + 7) // 8 * 8 + 32
    return min(stored, total(fixed), total(dyn)) // 8


def chain_sizes(d: bytes, minmatch: int, too_far: int) -> dict:
    a = np.frombuffer(d, np.uint8)
    nseg = (len(d) + dr.SEGMENT - 1) // dr.SEGMENT
    best = ch.best_all(d, DEPTHS, minmatch, too_far)
    out = {}
    for depth in DEPTHS:
        L, O = (x.tolist() for x in best[depth])
        for lazy, margin in itertools.product(LAZIES, MARGINS):
            tot = 0
            for k in range(nseg):
                lo, hi = k * dr.SEGMENT, min(len(d), (k + 1) * dr.SEGMENT)
                seqs = [(m - lo, l, o) for m, l, o in ch.parse(L, O, lo, hi, lazy, margin)]
                tot += segment_bytes(a[lo:hi], seqs, k + 1 == nseg)
            out[(minmatch, too_far, depth, lazy, margin)] = tot / len(d)
    return out


def baseline_sizes(d: bytes) -> dict:
    segs = [d[k:k + dr.SEGMENT] for k in range(0, len(d), dr.SEGMENT)]
    out = {"greedy": len(dr.deflate(d)) / len(d)}
    for lvl in (1, 4, 6):
        tot = 0
        for s in segs:
            c = zlib.compressobj(lvl, zlib.DEFLATED, -15)
            tot += len(c.compress(s) + c.flush())
        out[f"zlib -{lvl}"] = tot / len(d)
    return out


def job(arg):
    name, mib, what = arg
    d = corpus(name, mib << 20)
    res = baseline_sizes(d) if what == "base" else chain_sizes(d, *what)
    return (name, mib), res


def check(name: str):
    d = corpus(name, 1 << 20)
    for mm, tf in MATCH_RULES:
        got = chain_sizes(d, mm, tf)[(mm, tf, 16, 2, 4)]
        want = len(ch.deflate(d, depth=16, lazy=2, margin=4, minmatch=mm, too_far=tf)) / len(d)
        assert got == want, (name, mm, tf, got, want)
    print(f"check {name}: histogram sizes equal the encoded streams", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8")
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    names = ["text", "binary", "repeated", "half-zero"]
    if args.check:
        for nm in names:
            check(nm)
    cols = [(nm, int(s)) for s in args.sizes.split(",") for nm in names]
    work = [(nm, mib, w) for nm, mib in cols for w in ["base", *MATCH_RULES]]
    work.sort(key=lambda x: -x[1])
    table = {c: {} for c in cols}
    with Pool(args.jobs) as p:
        for col, res in p.imap_unordered(job, work):
            table[col].update(res)
    rows = ["greedy", "zlib -1", "zlib -4", "zlib -6"] + sorted(k for k in table[cols[0]] if isinstance(k, tuple))
    print("| row (MINMATCH, TOO_FAR, DEPTH, LAZY, MARGIN) | " + " | ".join(f"{nm} {mib} MiB" for nm, mib in cols) + " |")
    print("|---" * (len(cols) + 1) + "|")
    for r in rows:
        print(f"| {r if isinstance(r, str) else '(' + ', '.join(map(str, r)) + ')'} | "
              + " | ".join(f"{table[c][r]:.4f}" for c in cols) + " |")


if __name__ == "__main__":
    main()
