"""Pins the multi-block XZ cases (tests/xz_block_cases.py) on the CPU: every status is the oracle's, every valid archive decodes
to the same bytes through liblzma, the backward walk finds exactly the forward walk's blocks on every valid archive, and on
every case built for the two walks to disagree it finds block starts or sizes the forward walk does not."""
import pytest

import xz_block_cases as XB
import xz_cases as X

DISAGREE = ("swapped", "record count", "one record too few", "cut at the look-alike", "look-alike stream behind")


def test_statuses_match_oracle(oracle):
    bad = [(a.name, oracle.xz_unarchive(a.data)[0], a.status) for a in XB.cases() if oracle.xz_unarchive(a.data)[0] != a.status]
    assert not bad, bad


def test_valid_cases_decode_through_liblzma(oracle):
    valid = [a for a in XB.cases() if a.status == X.OK]
    assert len(valid) > 20
    for a in valid:
        assert XB.liblzma(a.data) == oracle.xz_unarchive(a.data)[1], a.name


def test_walks_agree_on_valid_cases(oracle):
    for a in XB.cases() + [c for c in X.cases() if c.status == X.OK and c.data]:
        if a.status != X.OK:
            continue
        back = XB.back_walk(a.data)
        assert back is not None, a.name
        assert [(s, n) for s, n, _ in back] == XB.forward_blocks(a.data), a.name
        out = oracle.xz_unarchive(a.data)[1]
        assert sum(n for _, n, _ in back) == len(out), a.name


@pytest.mark.parametrize("name", [a.name for a in XB.cases() if a.name.startswith(("unpadded", "decoded", "record", "one record",
                                                                                     "cut at", "look-alike stream"))])
def test_disagreement_cases_differ(name):
    a = [c for c in XB.cases() if c.name == name][0]
    back = XB.back_walk(a.data)
    fwd = XB.forward_blocks(a.data)
    assert back is None or [(s, n) for s, n, _ in back] != fwd, (name, back, fwd)


def test_catalogue_shape():
    names = [a.name for a in XB.cases()]
    assert "64 blocks, sizes True" in names and "stream of zero blocks" in names
    assert sum(n.startswith(DISAGREE) or "swapped" in n for n in names) >= 7
    arc, cut = XB.lookalike()
    back = XB.back_walk(arc[:cut])
    assert back is not None and back[0][0] == 12          # the look-alike covers the cut unit from byte 0
