"""Restatement of the compressed DataBlob format whose Huffman literals cover every byte value
(pbsgpu_blob_encode_batch_lzh, K10 with its full-alphabet flag in csrc/zent.cu) in numpy / pure Python.  Test
infrastructure: the GPU output is compared with it byte for byte, and libzstd's decoder checks it
(tests/test_zstd_huf_cpu.py).  The parse, the sequences section, the FSE table construction and the Huffman code are
tests/zstd_lz_ref.py's and tests/zstd_ent_ref.py's, unchanged.

The one change against _lze is the literals section: a block with >= 2 literal values may be Huffman-coded whatever its
largest value, because the tree description may also take zstd's FSE-compressed weight form (RFC 8878 4.2.1.2).  Per
block that is not constant, the Block_Content is the smallest of compressed_block (_lz), zstd_ent_ref.entropy_block
(_lze) and entropy_block_lzh below, the earlier one on ties; the block stays raw when none is smaller than the block.
So every _lzh blob is at most its _lze blob."""
from __future__ import annotations

import numpy as np

from oracle.pyref import BLOB_MAGIC_COMPRESSED, BLOB_MAGIC_UNCOMPRESSED, ZFRAME_BLOCK
from zstd_ent_ref import (_Bits, _lit_header, HUF_MAXBITS, HUF_MAXSYMBOL, accuracy_log, entropy_block, fse_description,
                          huf_codes, huf_lengths, huf_stream, normalize, sequences_section)
from zstd_lz_ref import LZ_HBITS, LZ_MINMATCH, LZ_TILE, compressed_block, fse_table, lz_parse

WEIGHT_MAXLOG = 6       # the largest accuracy log of the FSE table of Huffman weights (RFC 8878 4.2.1.2)
FSE_TREE_MAX = 127      # the FSE form's header byte is the compressed size, and must stay below 128


# -- tree descriptions -------------------------------------------------------------------------------------------------
def fse_weights(wts) -> bytes | None:
    """FSE-compressed weights (without the header byte): the table description of the weights' own distribution
    (accuracy log accuracy_log(len, distinct, 6)), then a bitstream of two interleaved states: the decoder reads
    state 1's start, then state 2's, then takes a weight from state 1, state 2, state 1, ... and stops when a state
    update reads past the start of the stream.  So state 1 codes the weights at even positions and state 2 those at
    odd ones; the encoder runs from the last weight to the first.

    Each state starts in the lowest state of its weight (zstd's FSE_initCState2), where the decoder's update reads at
    least one bit: the update after the second-to-last weight must run past the stream's start for the decoder to stop
    there.  (The "no bits written" start enc[code][0] reads no bits when the weight holds more than half of the states,
    as the zero weight often does.)  None when the form cannot state the list: fewer than 2 weights or 1 distinct value."""
    n = len(wts)
    counts = np.bincount(np.asarray(wts, np.int64), minlength=HUF_MAXBITS + 1).tolist()
    distinct = sum(1 for c in counts if c)
    if n < 2 or distinct < 2:
        return None
    log = accuracy_log(n, distinct, WEIGHT_MAXLOG)
    norm = normalize(counts, log)
    sym, nb, base, enc = fse_table(norm, log)
    first = {s: sym.index(s) for s in set(wts)}
    st = [first[wts[n - 2 + (n % 2)]], first[wts[n - 1 - (n % 2)]]]    # state 1: last even position; state 2: odd
    w = _Bits()
    for k in range(n - 3, -1, -1):
        t = k & 1
        u = enc[wts[k]][st[t]]
        w.add(st[t] - base[u], nb[u])
        st[t] = u
    w.add(st[1], log); w.add(st[0], log); w.add(1, 1)
    return fse_description(norm, log) + w.flush()


def tree_description(lengths) -> bytes | None:
    """Huffman tree description of the code lengths: the weights (maxbits + 1 - length, or 0) of symbols 0..top-1; the
    weight of `top`, the largest present symbol, is implied.  Of the two forms the smaller one that is allowed, the
    direct one on ties; None when neither is:
      direct  header byte 127 + top, then the weights 4 bits each, two per byte, the first in the high nibble; top <= 128
      FSE     header byte = the size of fse_weights (< 128), then fse_weights"""
    mx, top = max(lengths), max(s for s in range(len(lengths)) if lengths[s])
    wts = [mx + 1 - lengths[s] if lengths[s] else 0 for s in range(top)]
    forms = []
    if top <= HUF_MAXSYMBOL:
        w2 = wts + [0]
        forms.append(bytes([127 + top]) + bytes(w2[k] << 4 | w2[k + 1] for k in range(0, top, 2)))
    fse = fse_weights(wts)
    if fse is not None and len(fse) <= FSE_TREE_MAX:
        forms.append(bytes([len(fse)]) + fse)
    return min(forms, key=len) if forms else None


# -- literals ----------------------------------------------------------------------------------------------------------
def huffman_literals_tree(lits: np.ndarray, lengths, tree: bytes) -> bytes:
    """Compressed_Literals_Block with the given tree description: zstd_ent_ref.huffman_literals's streams, stream count
    and Size_Format rule."""
    codes = np.array(huf_codes(lengths), np.int64)
    ln_arr = np.array(lengths, np.int64)
    n = len(lits)
    one = tree + huf_stream(lits, codes, ln_arr)
    if n <= 1023 and len(one) <= 1023:
        return (2 | n << 4 | len(one) << 14).to_bytes(3, "little") + one
    seg = (n + 3) // 4
    st = [huf_stream(lits[k * seg:min(n, (k + 1) * seg)], codes, ln_arr) for k in range(4)]
    body = tree + b"".join(len(s).to_bytes(2, "little") for s in st[:3]) + b"".join(st)
    c = len(body)
    if max(n, c) <= 1023:
        return (2 | 1 << 2 | n << 4 | c << 14).to_bytes(3, "little") + body
    if max(n, c) <= 16383:
        return (2 | 2 << 2 | n << 4 | c << 18).to_bytes(4, "little") + body
    return (2 | 3 << 2 | n << 4 | c << 22).to_bytes(5, "little") + body


def literals_section_lzh(lits: bytes) -> bytes:
    """RLE_Literals_Block when all literals have one value; Huffman-coded when there are >= 2 values, a tree form is
    allowed, and that section is smaller than the raw one; else Raw_Literals_Block."""
    raw = _lit_header(0, len(lits)) + lits
    if not lits:
        return raw
    a = np.frombuffer(lits, np.uint8)
    hist = np.bincount(a, minlength=256).tolist()
    if np.count_nonzero(hist) == 1:
        return _lit_header(1, len(lits)) + lits[:1]
    lengths = huf_lengths(hist)
    tree = tree_description(lengths)
    if tree is None:
        return raw
    huf = huffman_literals_tree(a, lengths, tree)
    return huf if len(huf) < len(raw) else raw


def entropy_block_lzh(lits: bytes, seqs) -> bytes:
    """Block_Content with the full-alphabet literals: literals_section_lzh + sequences_section."""
    return literals_section_lzh(bytes(lits)) + sequences_section(seqs)


def block_content_lzh(lits: bytes, seqs) -> bytes:
    """The smallest of the _lz content, the _lze content and entropy_block_lzh, the earlier one on ties."""
    return min((compressed_block(lits, seqs), entropy_block(lits, seqs), entropy_block_lzh(lits, seqs)), key=len)


def zstd_frame_lzh(data: bytes, hbits: int = LZ_HBITS, tile: int = LZ_TILE, minmatch: int = LZ_MINMATCH) -> bytes:
    """zstd_ent_ref.zstd_frame_lze's frame with block_content_lzh: every block is at most its _lze block."""
    data = bytes(data)
    out = bytearray(b"\x28\xb5\x2f\xfd\xe0" + len(data).to_bytes(8, "little"))
    nb = max(1, (len(data) + ZFRAME_BLOCK - 1) // ZFRAME_BLOCK)
    for b in range(nb):
        blk = data[b * ZFRAME_BLOCK:(b + 1) * ZFRAME_BLOCK]
        last = int(b + 1 == nb)
        if len(blk) > 0 and blk.count(blk[:1]) == len(blk):
            out += (last | 1 << 1 | len(blk) << 3).to_bytes(3, "little") + blk[:1]
            continue
        body = block_content_lzh(*lz_parse(blk, hbits, tile, minmatch)) if blk else blk
        if len(body) < len(blk):
            out += (last | 2 << 1 | len(body) << 3).to_bytes(3, "little") + body
        else:
            out += (last | len(blk) << 3).to_bytes(3, "little") + blk
    return bytes(out)


def blob_encode_lzh(data: bytes) -> bytes:
    """blob_encode with zstd_frame_lzh as the compressed payload (kept only when smaller than the raw bytes)."""
    import zlib
    data = bytes(data)
    if data:
        fr = zstd_frame_lzh(data)
        if len(fr) < len(data):
            return BLOB_MAGIC_COMPRESSED + zlib.crc32(fr).to_bytes(4, "little") + fr
    return BLOB_MAGIC_UNCOMPRESSED + zlib.crc32(data).to_bytes(4, "little") + data


# -- test data ---------------------------------------------------------------------------------------------------------
def binary_corpus(nbytes: int, seed: int = 0) -> np.ndarray:
    """Deterministic binary-like test data: interleaved 4-32 KiB stretches of
      - an instruction-like stream: a Zipf-drawn vocabulary of 1-15-byte sequences that start with an opcode byte (most
        of them >= 0x80) followed by ModRM-like and small immediate bytes, a third of them followed by a random 32-bit
        displacement (small, or any value);
      - tables of little-endian uint32 with small deltas;
      - float32 arrays of a smooth signal (a sum of two sines)."""
    rng = np.random.default_rng(seed)
    ops = np.array([0x48, 0x89, 0x8B, 0xE8, 0xFF, 0x0F, 0x83, 0xC3, 0x85, 0x74, 0x75, 0xEB, 0xC7, 0x8D, 0x31, 0x39,
                    0x41, 0x4C, 0x80, 0x84, 0x88, 0xB8, 0xBE, 0xBF, 0xC1, 0xD1, 0xE9, 0xF6, 0xF7, 0x66, 0x90, 0xCC],
                   np.uint8)
    body = np.concatenate([np.arange(0x40, 0xC0, 8), [0, 0, 0, 0, 1, 2, 4, 8, 0x10, 0x20, 0xFF, 0xFF]]).astype(np.uint8)
    vocab = []
    for _ in range(2048):
        ln = int(min(15, 1 + rng.geometric(0.3)))
        vocab.append(np.concatenate([[rng.choice(ops)], rng.choice(body, ln - 1)]).astype(np.uint8))
    vflat = np.concatenate(vocab)
    vlen = np.array([len(v) for v in vocab], np.int64)
    vstart = np.concatenate([[0], np.cumsum(vlen)[:-1]])
    p = 1.0 / np.arange(1, len(vocab) + 1) ** 1.1
    p /= p.sum()
    out = np.empty(nbytes, np.uint8)
    pos = 0
    while pos < nbytes:
        want = min(int(rng.integers(4, 33)) << 10, nbytes - pos)
        kind = rng.choice(3, p=[0.6, 0.2, 0.2])
        if kind == 0:
            m = want // 3 + 16
            ids = rng.choice(len(vocab), m, p=p)
            disp = rng.random(m) < 0.33
            big = rng.random(m) < 0.5
            val = np.where(big, rng.integers(0, 1 << 32, m), rng.integers(-4096, 4096, m) & 0xFFFFFFFF)
            dbytes = val.astype("<u4").view(np.uint8).reshape(m, 4)
            L = vlen[ids] + 4 * disp
            ends = np.cumsum(L)
            src = np.repeat(vstart[ids] - (ends - L), L) + np.arange(int(ends[-1]))
            tail = np.arange(int(ends[-1])) - np.repeat(ends - L + vlen[ids], L)   # >= 0: byte of the displacement
            inst = tail < 0
            seg = np.empty(int(ends[-1]), np.uint8)
            seg[inst] = vflat[src[inst]]
            owner = np.repeat(np.arange(m), L)
            seg[~inst] = dbytes[owner[~inst], tail[~inst]]
            seg = seg[:want]
        elif kind == 1:
            n = (want + 3) // 4
            v = int(rng.integers(0, 1 << 24)) + np.cumsum(rng.integers(0, 64, n))
            seg = (v & 0xFFFFFFFF).astype("<u4").view(np.uint8)[:want]
        else:
            n = (want + 3) // 4
            t = np.arange(n) * rng.uniform(0.001, 0.02)
            v = rng.uniform(1, 1000) * np.sin(t) + rng.uniform(0.1, 10) * np.sin(7.3 * t + 1.0)
            seg = v.astype("<f4").view(np.uint8)[:want]
        out[pos:pos + len(seg)] = seg
        pos += len(seg)
    return out
