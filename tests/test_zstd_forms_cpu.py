"""The block-form census (tests/zstd_forms.py) on the CPU: the frame walker reads back what the restatements decided,
every form_cases() chunk reaches the forms it is built for under each mode's restatement, libzstd decodes every frame,
and the census of the GPU test inputs plus form_parts() covers REQUIRED[mode] for every mode."""
import numpy as np
import pytest

from oracle import pyref
import zstd_ent_ref as entref
import zstd_forms as zf
import zstd_huf_ref as hufref
import zstd_lz_ref as lzref

pa = pytest.importorskip("pyarrow")
B = pyref.ZFRAME_BLOCK
FRAME = {"lz": lzref.zstd_frame_lz, "lze": entref.zstd_frame_lze, "lzh": hufref.zstd_frame_lzh}


def decode(frame: bytes, size: int) -> bytes:
    return pa.Codec("zstd").decompress(frame, decompressed_size=size).to_pybytes() if size else b""


def gpu_inputs():
    """Every input of the GPU zstd and encrypted-blob tests but the chunker-output images."""
    from test_gpu_zstd_ent import entropy_parts
    from test_gpu_zstd_huf import binary_parts
    from test_gpu_zstd_lz import mixed_parts
    return mixed_parts() + entropy_parts() + binary_parts()


@pytest.fixture(scope="module")
def frames():
    """mode -> (parts, their restatement frames): form_parts() first, then the GPU test inputs."""
    parts = zf.form_parts() + gpu_inputs()
    return {m: (parts, [FRAME[m](p.tobytes()) for p in parts]) for m in zf.MODES}


def expected(mode: str, blk: bytes, info: zf.BlockInfo):
    """What the restatement decided for a compressed block, re-derived from its parse and its table rules."""
    lits, seqs = lzref.lz_parse(blk)
    assert info.nseq == len(seqs) and info.lit_regen == len(lits)
    if info.lit_type == 2:
        hist = np.bincount(np.frombuffer(lits, np.uint8), minlength=256).tolist()
        lengths = entref.huf_lengths(hist)
        assert mode != "lz" and info.huf_maxlen == max(lengths)
        top = max(s for s in range(256) if lengths[s])
        assert info.tree_weights == top
        tree = hufref.tree_description(lengths) if mode == "lzh" else None
        if tree is not None and tree[0] < 128:
            assert info.tree == "fse"
            wts = [max(lengths) + 1 - ln if ln else 0 for ln in lengths[:top]]
            assert info.tree_log == entref.accuracy_log(top, len(set(wts)), hufref.WEIGHT_MAXLOG)
        else:
            assert info.tree == "direct"
    else:
        assert info.lit_type == 0
    if not seqs:
        assert info.modes is None
        return
    if info.modes == (0, 0, 0):                                       # the _lz content
        assert info.logs == (None, None, None)
        return
    assert mode != "lz"
    codes = [lzref.seq_codes(*s) for s in seqs]
    for k, (col, nsym, cap) in enumerate(((0, 36, entref.LL_MAXLOG), (2, 32, entref.OF_MAXLOG),
                                          (1, 53, entref.ML_MAXLOG))):
        m, _, _, log = entref.table_for([c[col][0] for c in codes], nsym, cap)
        assert info.modes[k] == m and info.logs[k] == (log if m == 2 else None), (k, info)


@pytest.mark.parametrize("mode", zf.MODES)
def test_walker_reads_back_the_restatements_decisions(frames, mode):
    """Per block: type and size, literal type and count, Huffman code length, tree form and weight-table log,
    sequence count, column modes and logs; and libzstd decodes every frame."""
    parts, frs = frames[mode]
    n_checked = 0
    for p, fr in zip(parts, frs):
        data = p.tobytes()
        assert decode(fr, len(data)) == data
        infos = zf.walk(fr)
        assert len(infos) == max(1, (len(data) + B - 1) // B) and infos[-1].last
        for k, info in enumerate(infos):
            blk = data[k * B:(k + 1) * B]
            if info.type == 1:
                assert len(set(blk)) == 1 and info.size == len(blk)
            elif info.type == 0:
                assert info.size == len(blk)
            else:
                assert info.size < len(blk)
                expected(mode, blk, info)
                n_checked += 1
    assert n_checked > 50


@pytest.mark.parametrize("mode", zf.MODES)
def test_form_cases_reach_their_forms(mode):
    for i, (p, want) in enumerate(zf.form_cases()):
        got = zf.census([FRAME[mode](p.tobytes())])
        assert want.get(mode, set()) <= set(got), (i, sorted(want.get(mode, set()) - set(got)))


def test_form_case_premises():
    """What the recipes promise beyond the forms: every word after the first tile is one 4-byte match, the Fibonacci
    literals need the length limit, and the two-value chunk has no earlier tile."""
    words = zf.word_block()
    lits, seqs = lzref.lz_parse(words.tobytes())
    assert len(seqs) == 32704 and lits == words[:256].tobytes() and {s[1] for s in seqs} == {4}
    fib = zf.fib_symbols()
    lits, _ = lzref.lz_parse(fib.tobytes())
    hist = np.bincount(np.frombuffer(lits, np.uint8), minlength=256).tolist()
    assert len(lits) > 16383 and max(lits) <= entref.HUF_MAXSYMBOL
    assert max(entref._huffman(hist)) > entref.HUF_MAXBITS
    assert entref.literals_section(lits)[0] & 3 == 2                 # the Huffman section is what gets written
    period = zf.mutated_period()
    _, seqs = lzref.lz_parse(period.tobytes())
    assert {s[2] for s in seqs} == {600}


@pytest.mark.parametrize("mode", zf.MODES)
def test_census_covers_the_required_forms(frames, mode):
    parts, frs = frames[mode]
    c = zf.census(frs)
    print(f"\n{mode} census:")
    for name in sorted(c):
        print(f"  {name:24s} {c[name]:6d}{'  (required)' if name in zf.REQUIRED[mode] else ''}")
    assert not zf.REQUIRED[mode] - set(c), sorted(zf.REQUIRED[mode] - set(c))
