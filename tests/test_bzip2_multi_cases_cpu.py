"""The multi-stream catalogue (tests/bzip2_multi_cases.py) pinned on the CPU: every case's status is what the oracle's
BZip2.multiDecompress returns, valid files decode as Python's bz2 decodes them, and the byte cuts of the three-stream file
cover the statuses a cut can give."""
import bz2

import bzip2_multi_cases as M


def test_statuses_match_oracle(oracle):
    bad = []
    for c in M.cases():
        st, parts, whole = oracle.bzip2_multi_decompress(c.data)
        if st != c.status:
            bad.append((c.name, st, c.status))
    assert not bad


def test_valid_cases_match_bz2(oracle):
    for c in M.cases():
        if c.status != M.OK:
            continue
        st, whole, ends, starts = M.expect(oracle, c.data)
        if c.libbz2:
            assert whole == (bz2.decompress(c.data) if c.data else b""), c.name
        assert len(ends) == len(starts) and starts[:1] == ([0] if c.data else [])


def test_wrong_crc_payload_is_the_failing_stream(oracle):
    for c in M.cases():
        if c.status != M.WRONG_CRC:
            continue
        st, whole, ends, starts = M.expect(oracle, c.data)
        assert st == M.WRONG_CRC and len(ends) >= 1 and ends[-1] == len(whole), c.name


def test_three_stream_cuts_cover_the_statuses(oracle):
    seen = {oracle.bzip2_multi_decompress(d)[0] for _, d in M.cuts()}
    assert {M.OK, M.WRONG_MAGIC} <= seen and len(seen) >= 3
