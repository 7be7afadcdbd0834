"""The read side of encrypt mode without a GPU: the status the header adds for a failed GCM tag has the value the
bindings use, and the new call is declared with the plain call's arguments after the crypt handle."""
import re
from pathlib import Path

from pbs_plus_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent


def test_bad_tag_follows_the_decode_statuses():
    hdr = (ROOT / "include" / "pbsgpu.h").read_text()
    assert re.search(r"enum \{ PBSGPU_DEC_BAD_TAG = PBSGPU_DEC_BAD_DIGEST \+ 1 \};", hdr)
    assert _lib.DEC_BAD_TAG == _lib.DEC_BAD_DIGEST + 1 == 8


def test_decode_enc_takes_the_plain_arguments_after_the_crypt_handle():
    hdr = " ".join((ROOT / "include" / "pbsgpu.h").read_text().split())
    args = lambda name: re.search(name + r"\(pbsgpu_ctx \*ctx, (.*?)\);", hdr).group(1)
    plain, enc = args(r"int pbsgpu_blob_decode_batch"), args(r"int pbsgpu_blob_decode_batch_enc")
    assert enc == "const pbsgpu_crypt *crypt, " + plain
