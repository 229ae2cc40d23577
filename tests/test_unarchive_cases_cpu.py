"""Pins the unarchive catalogue (tests/unarchive_cases.py) against the CPU oracle before any GPU runs: every archive's stated
status, payload and consumed byte count must be the oracle's gzip_unarchive / zlib_unarchive answer."""
import pytest

import unarchive_cases as U


@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_catalogue_matches_oracle(oracle, fmt):
    arcs = [a for a in U.cases() if a.fmt == fmt]
    names = [a.name for a in arcs]
    assert len(set(names)) == len(names)
    bad = []
    for a in arcs:
        st, out, used = U.oracle_unarchive(oracle, fmt, a.data)
        if a.status is not None and st != a.status:
            bad.append((a.name, "status", st, a.status))
        elif a.payload is not None and (st not in (U.OK,) + U.PAYLOAD_CARRYING or out != a.payload):
            bad.append((a.name, "payload", st))
        elif a.consumed is not None and used != a.consumed:
            bad.append((a.name, "consumed", used, a.consumed))
    assert not bad, f"{len(bad)} of {len(arcs)} archives differ from the oracle: {bad[:10]}"


def test_catalogue_covers_every_kind():
    arcs = U.cases()
    stated = {a.status for a in arcs}
    for st in (U.OK, U.GZ_MAGIC, U.GZ_METHOD, U.GZ_FLAGS, U.GZ_HCRC, U.GZ_CRC, U.GZ_ISIZE, U.TRAP, U.ZL_METHOD, U.ZL_CINFO,
               U.ZL_FCHECK, U.ZL_ADLER, U.WRONG_BLOCK_TYPE, 101, 103, 104):
        assert st in stated, st
    assert sum(a.name.startswith("gzip header ") for a in arcs) == len(U.GZIP_CASES)
    assert sum(a.name.startswith("zlib header ") for a in arcs) == len(U.ZLIB_CASES)
