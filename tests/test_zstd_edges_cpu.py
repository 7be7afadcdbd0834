"""The blob decoder's edge frames without a GPU: every case of tests/zstd_edge_frames.py gets the verdict upstream's
streaming libzstd decoder gives it (the content for a valid case, a refusal for an invalid one) but for the
KNOWN_DIFFERENCES, where both verdicts are pinned; the cases reach every edge in zstd_forms.REQUIRED_EDGES, measured from
their bytes, and each case reaches one that no other case does; and the RFC decoder that measures them agrees with
libzstd on the fixture and on libzstd's own frames."""
from collections import Counter

import pytest

import zstd_dec_forms as zd
import zstd_edge_frames as ef
import zstd_forms as zf
import zstd_stream_ref as sr
from pbs_plus_b200 import _lib


@pytest.fixture(scope="module")
def libzstd():
    sr.require()
    return sr


def test_every_case_gets_the_streaming_libzstd_verdict(libzstd):
    cases = ef.edge_cases()
    assert len({c.name for c in cases}) == len(cases)
    for c in cases:
        got = libzstd.stream_decode(c.payload)
        if c.name in ef.KNOWN_DIFFERENCES:
            continue
        if c.content is None:
            assert isinstance(got, str), (c.name, len(got))
        else:
            assert got == c.content, (c.name, got if isinstance(got, str) else len(got))
            assert c.status == _lib.DEC_OK and c.size == len(c.content)


def test_known_differences_pin_both_verdicts(libzstd):
    """libzstd 1.5.5 reads these, the RFC decoder and K13 refuse them; a change on either side fails here."""
    cases = {c.name: c for c in ef.edge_cases()}
    assert libzstd.version() == "1.5.5", "the table was written against libzstd 1.5.5; check each entry again"
    for name, (size, why) in ef.KNOWN_DIFFERENCES.items():
        c = cases[name]
        got = libzstd.stream_decode(c.payload)
        assert isinstance(got, bytes) and len(got) == size, (name, got if isinstance(got, str) else len(got))
        assert c.content is None and c.status == _lib.DEC_BAD_FRAME and why
        with pytest.raises(zf.Reject):
            zf.decode_payload(c.payload)


def case_forms() -> dict[str, set]:
    """The edges each case reaches, read from its bytes; an invalid case adds the rule it breaks."""
    out = {}
    for c in ef.edge_cases():
        forms = Counter()
        try:
            got = zf.decode_payload(c.payload, forms)
            assert c.content is not None and got == c.content, c.name
        except zf.Reject as e:
            assert c.content is None, (c.name, e.rule)
            forms[f"reject:{e.rule}"] += 1
        out[c.name] = {f for f, k in forms.items() if k}
    return out


def test_the_cases_reach_every_required_edge_and_each_case_one_of_its_own():
    per_case = case_forms()
    seen = Counter(f for forms in per_case.values() for f in forms)
    print("\nedge census:")
    for form, k in sorted(seen.items()):
        print(f"  {form:28s} {k}")
    missing = zf.REQUIRED_EDGES - set(seen)
    assert not missing, missing
    # so removing any case from the builder loses an edge
    for name, forms in per_case.items():
        own = {f for f in forms & zf.REQUIRED_EDGES if seen[f] == 1}
        assert own, f"{name} reaches no required edge of its own: {sorted(forms)}"


def test_the_census_decoder_agrees_with_libzstd_on_the_fixture_and_libzstd_frames(libzstd):
    pytest.importorskip("pyarrow")
    from test_zstd_decode_cpu import libzstd_payloads
    payloads = [p for p, _ in zd.fixture_cases().values()]
    payloads += [p for _, _, p, _ in libzstd_payloads(1 << 18, 2)]
    for k, p in enumerate(payloads):
        want = libzstd.stream_decode(p)
        assert isinstance(want, bytes), k
        assert zf.decode_payload(p) == want, k


def test_the_census_decoder_refuses_truncations_libzstd_refuses(libzstd):
    """Every cut of a small multi-frame payload (blocks, a skippable frame, a checksum) is refused by both."""
    case = {c.name: c for c in ef.edge_cases()}["checksum_unaligned"]
    payload = case.payload + ef.skippable(3) + {c.name: c for c in ef.edge_cases()}["rep_reset"].payload
    assert zf.decode_payload(payload) == libzstd.stream_decode(payload)
    ends, pos = set(), 0
    for _, fr in zd.split_payload(payload):
        pos += len(fr)
        ends.add(pos)
    for cut in range(1, len(payload)):
        if cut in ends:                                          # a cut between frames leaves a complete payload
            continue
        assert isinstance(libzstd.stream_decode(payload[:cut]), str), cut
        with pytest.raises(zf.Reject):
            zf.decode_payload(payload[:cut])
