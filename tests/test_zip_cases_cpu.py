"""The hand-built ZIP catalogue (zip_cases.py) on the CPU: the oracle's ZipContainer.open / info and the engine's host-side
swc_zip_info against the expectations derived from the Swift source, the writer's traces against what each family claims
to exercise, zipfile on the well-formed cases, and every byte truncation through the oracle."""
import io
import zipfile

import pytest

import zip_cases as Z

CASES = Z.cases()
IDS = [c.name for c in CASES]
FIELDS = ("name", "data", "crc", "size", "method", "is_directory", "utf8")


def strip(ents):
    return [{k: e[k] for k in FIELDS} for e in ents]


def test_catalogue_names_are_unique():
    assert len(set(IDS)) == len(IDS)


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_oracle_open_and_info_match_expectation(oracle, c):
    st, ents = oracle.zip_open(c.blob)
    assert st == c.status
    assert strip(ents) == c.entries
    st, ents = oracle.zip_open(c.blob, info_only=True)
    assert st == c.info_status
    assert strip(ents) == c.info_entries


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_engine_info_matches_expectation(c):
    import swcompression_b200 as S
    from swcompression_b200.api import _zip_text
    try:
        infos, st = S.ZipContainer.info(c.blob), 0
    except S.SWCompressionError as e:
        infos, st = [], e.code
    assert st == c.info_status
    assert [(i.name, i.size, i.crc, i.type == "directory") for i in infos] == \
        [(_zip_text(w["name"], w["utf8"]), w["size"], w["crc"], w["is_directory"]) for w in c.info_entries]


def _family(n):
    return [c for c in CASES if c.family == n]


def test_extra_field_steps_land_on_the_data():
    """the reader offset after the last extra field, summed from the steps each case states for its fields, is where the
    writer put the entry data (local) or the file comment (central); and the families reach the rules they are named for"""
    seen = set()
    for c in _family(2):
        for t in c.built.trace:
            for where in ("local", "central"):
                tr = t.get(where)
                if not tr or not tr["fields"]:
                    continue
                assert tr["reader_end"] == tr["data_off"], (c.name, where)
                for id, declared, step, _ in tr["fields"]:
                    if id != Z.FILLER:
                        seen.add((where, id, declared != step))
    for rule in [("local", 0x000A, True), ("central", 0x000A, True), ("local", 0x7855, True), ("local", 0x7875, True),
                 ("central", 0x7875, True), ("local", 0x0001, True), ("central", 0x0001, True), ("local", 0x5455, False)]:
        assert rule in seen, rule


def test_families_reach_what_they_claim():
    tags = {n: set().union(*(c.tags for c in _family(n))) for n in range(1, 8)}
    assert {"lookalike", "zip64_end"} <= tags[1]
    assert {"zip64_local", "zip64_central"} <= tags[2]
    assert {"descriptor", "wide", "narrow", "second_decode"} <= tags[5]
    assert {"mid_byte", "lzma", "lzma_wide", "second_decode"} <= tags[6]
    assert {"crc", "second_decode"} <= tags[7]
    statuses = {c.status for c in CASES}
    for st in (Z.OK, Z.TRAP, Z.SIGNATURE, Z.SIZE, Z.VERSION, Z.VOLUMES, Z.METHOD, Z.CRC, Z.TEXT, Z.LZMA_PROPERTIES):
        assert st in statuses
    # every LZMA entry's realCompSize is 9 + what the decoder model consumed (the cases set compSize from it)
    lz = [c for c in _family(6) if c.name.startswith("lzma_lc")]
    assert len({c.name for c in lz if "lzma_wide" in c.tags}) >= 6
    # look-alikes: a signature other than the real record's where a probe can meet it (behind it in the comment, or in
    # front of it in entry data)
    look = [c for c in _family(1) if "lookalike" in c.tags]
    assert len(look) >= 2
    for c in look:
        at = [k for k in range(len(c.blob) - 21) if c.blob.startswith(b"PK\x05\x06", k)]
        assert any(k != c.built.eocd_off for k in at), c.name


def _well_formed(c):
    """zipfile is stricter than the reference about records it does not need (local names, overlaps, extra-field sizes,
    the archive extra data record) and reads the end records its own way: compare on the plainly well-formed cases"""
    return (c.status == Z.OK and c.engine is None and c.family in (1, 5, 6, 7) and not c.tags & {"lookalike", "zip64_end"}
            and "archive_extra" not in c.name and "overlapping" not in c.name and "shared" not in c.name
            and "local64" not in c.name and "last_21" not in c.name and "central_uncomp" not in c.name)


WELL_FORMED = [c for c in CASES if _well_formed(c)]


def test_the_well_formed_subset_is_not_empty():
    assert len(WELL_FORMED) >= 30


@pytest.mark.parametrize("c", WELL_FORMED, ids=lambda c: c.name)
def test_zipfile_reads_the_well_formed_cases(c):
    with zipfile.ZipFile(io.BytesIO(c.blob)) as z:
        infos = z.infolist()
        assert [i.filename.encode("utf-8" if i.flag_bits & 0x800 else "cp437") for i in infos] == [w["name"] for w in c.entries]
        for zi, w in zip(infos, c.entries):
            if w["is_directory"] or w["method"] not in (0, 8, 12):
                continue
            assert z.read(zi) == w["data"]


def test_every_truncation_of_small_cases_runs_through_the_oracle(oracle):
    n = 0
    for c in CASES:
        if len(c.blob) > 2048:
            continue
        for k in range(len(c.blob)):
            st, ents = oracle.zip_open(c.blob[:k])
            assert st == Z.OK or st > 0
            n += 1
    assert n > 10000
