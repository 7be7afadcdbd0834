"""The GPU zstd encoders (K9, K10; pbsgpu_blob_encode_batch_lz / _lze / _lzh and _enc) through every block form they
write: tests/zstd_forms.py's form_parts() equal the restatements byte for byte, libzstd decodes them, and the census of
the GPU's own frames covers REQUIRED[mode]; the same through the encrypted blob call; and one batch whose 32 704-sequence
blocks sit on both sides of the edge between two passes of LZ_PASS_BLOCKS blocks."""
import os

import pytest

import crypt_ref
from oracle import pyref
import zstd_forms as zf
import zstd_huf_ref as hufref
import zstd_ent_ref as entref
import zstd_lz_ref as lzref
import pbs_plus_b200 as pg
from test_gpu_zstd_lz import check_blob, pack, to_dev

pytestmark = pytest.mark.gpu
pa = pytest.importorskip("pyarrow")
B = pyref.ZFRAME_BLOCK
PASS_BLOCKS = 4096                      # LZ_PASS_BLOCKS in csrc/zlz.cuh
KEY = bytes(range(40, 72))
BLOB = {"lz": lzref.blob_encode_lz, "lze": entref.blob_encode_lze, "lzh": hufref.blob_encode_lzh}


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module", autouse=True)
def release_device_memory(torch):
    """The pass-edge batch's tensors go back to the device when the module is done, not into torch's cache: later
    modules need nearly all of the HBM free."""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def eng():
    e = pg.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def parts():
    from test_zstd_forms_cpu import gpu_inputs
    return zf.form_parts() + gpu_inputs()


def frames_of(blobs):
    return [b[12:] for b in blobs if b[:8] == pyref.BLOB_MAGIC_COMPRESSED]


@pytest.mark.parametrize("mode", zf.MODES)
def test_form_parts_equal_the_restatement_and_cover_the_required_forms(eng, torch, parts, mode):
    """form_parts() and the other GPU tests' inputs, host and device bases, ragged offsets: the census is of the GPU's
    frames, per form_parts() chunk and over the whole batch."""
    ref = [BLOB[mode](p.tobytes()) for p in parts]
    buf, off, ln = pack(parts, 11)
    for base in (buf, to_dev(torch, buf)):
        blobs, crc = getattr(eng, f"blob_encode_batch_{mode}")(base, off, ln)
        for i, (blob, p) in enumerate(zip(blobs, parts)):
            assert blob == ref[i], (mode, i, len(blob), len(ref[i]))
            check_blob(blob, p.tobytes(), int(crc[i]))
        c = zf.census(frames_of(blobs))
        assert not zf.REQUIRED[mode] - set(c), sorted(zf.REQUIRED[mode] - set(c))
        for i, (_, target) in enumerate(zf.form_cases()):
            got = zf.census(frames_of(blobs[i:i + 1]))
            assert target.get(mode, set()) <= set(got), (i, sorted(target.get(mode, set()) - set(got)))


def test_form_parts_through_the_encrypted_blob_call(eng, torch):
    """_enc in lzh mode: every blob equals the restatement; the decrypted frames reach each part's lzh forms."""
    ps = zf.form_parts()
    buf, off, ln = pack(ps, 3)
    iv = os.urandom(16 * len(ps))
    ref = [crypt_ref.blob_encode_enc(KEY, iv[16 * i:16 * i + 16], p.tobytes(), "lzh") for i, p in enumerate(ps)]
    c = eng.crypt(KEY)
    try:
        for base in (buf, to_dev(torch, buf)):
            blobs, crc = eng.blob_encode_batch_enc(c, "lzh", base, off, ln, iv)
            for i, (b, p) in enumerate(zip(blobs, ps)):
                assert b == ref[i], i
                assert int(crc[i]) == int.from_bytes(b[8:12], "little")
                pl, comp = crypt_ref.blob_decrypt(KEY, b)
                assert comp and pa.Codec("zstd").decompress(pl, decompressed_size=len(p)).to_pybytes() == p.tobytes()
                got = zf.census([pl])
                target = zf.form_cases()[i][1].get("lzh", set())
                assert target <= set(got), (i, sorted(target - set(got)))
    finally:
        c.close()


@pytest.mark.parametrize("mode", ["lz", "lzh"])
def test_a_batch_across_a_pass_edge(eng, torch, mode):
    """4 095 copies of one compressible 128 KiB block (non-constant blocks 0..4 094), then the 32 704-sequence block at
    non-constant block 4 095, the last of the first pass, and again at 4 096, the first of the second; then the other
    form_parts().  K9a's sequence scratch and K10's entropy scratch are indexed by block within the pass, the slots by
    block within the call: a block read from the wrong pass slot changes its blob."""
    filler = lzref.text_corpus(B, 90)
    cases = zf.form_cases()
    words = cases[0][0]
    assert len(words) == B and "nseq:3B" in cases[0][1][mode]
    ps = [filler] * (PASS_BLOCKS - 1) + [words, words] + [p for p, _ in cases[1:]]
    buf, off, ln = pack(ps, 7)
    dev = to_dev(torch, buf)
    del buf
    blobs, crc = getattr(eng, f"blob_encode_batch_{mode}")(dev, off, ln)
    del dev
    f_want = BLOB[mode](filler.tobytes())
    assert f_want[:8] == pyref.BLOB_MAGIC_COMPRESSED
    for k in range(PASS_BLOCKS - 1):
        assert blobs[k] == f_want, k
    check_blob(blobs[0], filler.tobytes(), int(crc[0]))
    w_want = BLOB[mode](words.tobytes())
    for k in (PASS_BLOCKS - 1, PASS_BLOCKS):
        assert blobs[k] == w_want, k
        check_blob(blobs[k], words.tobytes(), int(crc[k]))
        assert "nseq:3B" in zf.census([blobs[k][12:]])
    for k, p in enumerate(ps[PASS_BLOCKS + 1:], PASS_BLOCKS + 1):
        assert blobs[k] == BLOB[mode](p.tobytes()), k
