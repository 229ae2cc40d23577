"""Pins the XZ catalogue (tests/xz_cases.py) against the CPU oracle before any GPU runs: every archive's stated status must be
the oracle's xz_unarchive answer, and the catalogue must reach every kind of case it promises."""
import xz_cases as X


def test_catalogue_matches_oracle(oracle):
    arcs = X.cases()
    bad = []
    for a in arcs:
        st, out, _ = oracle.xz_unarchive(a.data)
        if a.status is not None and st != a.status:
            bad.append((a.name, st, a.status))
        if a.unsupported and st == X.UNSUPPORTED:
            bad.append((a.name, "the oracle refuses an archive only the batch should refuse"))
    assert not bad, f"{len(bad)} of {len(arcs)} archives differ from the oracle: {bad[:10]}"


def test_catalogue_covers_every_kind(oracle):
    arcs = X.cases()
    stated = {oracle.xz_unarchive(a.data)[0] for a in arcs}
    for st in (X.OK, X.XZ_MAGIC, X.XZ_FIELD, X.XZ_CHECK, X.XZ_PADDING, 803, 804, 806, 809, 401):
        assert st in stated, st
    assert sum(a.unsupported for a in arcs) == 3
    assert sum(a.name.startswith("framing ") for a in arcs) == len(list(X.xz_cases()))
    assert sum(a.name.startswith("framed lzma_cases ") for a in arcs) * 12 >= len(X.lzma2_blocks()) > 20
