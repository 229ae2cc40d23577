"""The catalogue of tests/lz4_frame_cases.py against the oracle: its lz4_decompress agrees with the writer's model of
LZ4.decompress(data:dictionary:dictionaryID:) on every case and every byte cut: status, bytes, consumed bytes."""
import lz4_frame_cases as F


def _differences(oracle, cases):
    bad = []
    for c in cases:
        st, out, used = oracle.lz4_decompress(c.data, c.dictionary, c.dict_id)
        if st != c.status or (st in F.PAYLOAD and (out != c.out or used != c.consumed)):
            bad.append((c.name, st, c.status, len(out), len(c.out), used, c.consumed))
    return bad


def test_catalogue_matches_oracle(oracle):
    cases = F.catalogue()
    assert len(cases) > 1500
    assert {c.status for c in cases} >= {F.W.OK, F.W.TRUNCATED, F.W.CORRUPTED, F.W.CHECKSUM, F.W.UNSUPPORTED}
    bad = _differences(oracle, cases)
    assert not bad, (len(bad), bad[:8])


def test_truncations_match_oracle(oracle):
    cuts = [c for c, _ in F.truncations()]
    assert len(cuts) > 10000
    bad = _differences(oracle, cuts)
    assert not bad, (len(bad), bad[:8])


def test_catalogue_covers_the_frame_layer():
    cases = F.catalogue()
    by_name = {c.name: c for c in cases}
    # the dictionary is dropped behind a skippable frame: the same frame decodes with it and fails without
    assert by_name["needs dict"].status == F.W.OK and by_name["skip then needs dict"].status == F.W.CORRUPTED
    assert by_name["dict id matches"].status == F.W.OK and by_name["skip then dict id"].status == F.W.CORRUPTED
    assert by_name["skip then id mismatch dropped"].status == F.W.OK and by_name["dict id differs"].status == F.W.CORRUPTED
    # the block's room check counts the checksum's four bytes
    assert all(c.status == F.W.TRUNCATED for c in cases if c.name.endswith("sound k-1 room for checksum missing"))
    # consumed stops at the first frame
    assert by_name["second frame behind"].consumed == by_name["trailing bytes"].consumed < len(by_name["second frame behind"].data)
    assert {c.n_blocks for c in cases if c.n_blocks is not None} >= {0, 1, 31, 32, 33, 64, 65, 1000}
