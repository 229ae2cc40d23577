"""The TAR catalogue against the CPU restatement (oracle/tar.c), tarfile's own reading of the archives it wrote, and the
restatement of Swift's Double(String) the host uses for PAX times."""
import io
import math
import tarfile

import pytest

import swco_tar
import tar_cases as T
from swcompression_b200.api import swift_double, tar_entry, tar_entry_info

CASES = T.cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_catalogue_statuses(case):
    cid, data, info, opn, fst, fmt, n = case
    got_n, ist, ost, gfmt, gfst, _ = swco_tar.walk(data)
    assert (ist, ost, gfst) == (info, opn, fst)
    if fst == T.OK:
        assert gfmt == fmt
    if n is not None:
        assert got_n == n


def _info(cid, k=0):
    data = dict((c[0], c[1]) for c in CASES)[cid]
    return tar_entry_info(data, swco_tar.walk(data)[5][k])


def test_tarint_quirks():
    assert _info("octal_12_digits_lose_last").size == 1
    i = _info("octal_leading_space_nul")
    assert i.size == 5 and i.permissions is None
    i = _info("octal_signs")
    assert (i.size, i.ownerID, i.groupID) == (1, -7, 0)
    i = _info("octal_space_terminated")
    assert (i.size, i.modificationTime) == (3, float(0o17))
    i = _info("octal_bad_digit")
    assert i.ownerID is None and i.permissions is None
    assert _info("base256_size").ownerID == 1 << 40
    i = _info("base256_negative")
    assert (i.modificationTime, i.ownerID) == (-86400.0, -1)
    assert _info("base256_overflow_mtime").modificationTime is None


def test_layout_and_resolution():
    i = _info("gnu_times")
    assert (i.accessTime, i.creationTime, i.ownerUserName) == (1600000000.0, 1500000000.0, "user")
    i = _info("pre_posix")
    assert i.ownerUserName is None and i.deviceMajorNumber is None and i.accessTime is None
    assert (_info("prefix", 0).name, _info("prefix", 1).name) == ("dir/f", "dir/g")
    assert _info("prefix_gnu_ignored").name == "f"
    i = _info("bad_utf8_name")
    assert i.name == b"a\xffb\xc3".decode("utf-8", "replace") and i.linkName == "�"
    types = [_info("types", k).type for k in range(11)]
    assert types == ["regular", "regular", "hardLink", "symbolicLink", "characterSpecial", "blockSpecial", "directory", "fifo",
                     "contiguous", "unknown", "unknown"]
    assert [_info("negative_moves_back", k).name for k in range(3)] == ["A", "C", "B"]
    assert _info("gnu_long_name").name == "n" * 300
    assert _info("gnu_long_name_unterminated").name == "m" * 100
    assert _info("gnu_long_link").linkName == "k" * 200
    assert (_info("long_name_resets", 0).name, _info("long_name_resets", 1).name) == ("n" * 120, "plain")
    i = _info("pax_local")
    assert (i.name, i.size, i.ownerID, i.groupID, i.modificationTime, i.accessTime, i.creationTime) == \
        ("päx/name", 3, 4294967296, -3, 1700000000.5, 1.25, -25.0)
    assert (i.ownerUserName, i.ownerGroupName, i.linkName, i.charset, i.comment) == ("pu", "pg", "lp", "ISO-IR 10646 2000 UTF-8", "c")
    assert i.unknownExtendedHeaderRecords == {"vendor.x": "y"}
    a, b = _info("pax_global_persists", 0), _info("pax_global_persists", 1)
    assert (a.name, a.comment, a.modificationTime, a.unknownExtendedHeaderRecords) == ("l1", "g1", 5.0, {"g.k": "2"})
    assert (b.name, b.comment, b.modificationTime, b.unknownExtendedHeaderRecords) == ("second", "g1", 5.0, {"g.k": "1"})
    assert _info("pax_sun_x").name == "sun"
    assert _info("pax_empty").unknownExtendedHeaderRecords == {}
    assert _info("one_file").unknownExtendedHeaderRecords is None
    assert _info("pax_negative_length").unknownExtendedHeaderRecords == {"k": ""}
    assert _info("pax_plus_length").unknownExtendedHeaderRecords == {"k": "abcd"}
    i = _info("pax_value_not_utf8_skipped")
    assert i.name == "good" and i.unknownExtendedHeaderRecords == {}
    i = _info("pax_int_overwritten_nil")
    assert (i.ownerID, i.size) == (9, 1)
    i = _info("pax_time_falls_through")
    assert (i.modificationTime, i.accessTime, i.creationTime) == (12.5, 16.0, 8.0)
    assert _info("pax_value_with_newline").comment == "two\nlines"


@pytest.mark.parametrize("cid", sorted(T.REFERENCE_FIELDS))
def test_reference_named_files(cid):
    """the assertions of the reference's TarTests.swift:72-370 on the restated files: open's entries (info's for
    test_big_num_field, whose data is cut away) and formatOf"""
    data = dict((c[0], c[1]) for c in CASES)[cid]
    n, ist, ost, fmt, fst, recs = swco_tar.walk(data)
    assert fst == 0 and fmt == T.REFERENCE_FORMATS[cid]
    use_info = cid == "test_big_num_field"
    assert (ist if use_info else ost) == 0
    entries = [tar_entry_info(data, r) if use_info else tar_entry(data, r) for r in recs]
    want = T.REFERENCE_FIELDS[cid]
    assert len(entries) == len(want)
    for e, w in zip(entries, want):
        info = e if use_info else e.info
        for k, v in w.items():
            got = e.data if k == "data" else getattr(info, k)
            assert (got is not None) if v == "*" else got == v, (k, got, v)


def test_open_sizes():
    data = dict((c[0], c[1]) for c in CASES)["pax_size_cuts_open"]
    e = tar_entry(data, swco_tar.walk(data)[5][0])
    assert e.data == b"hel" and e.info.size == 3
    data = dict((c[0], c[1]) for c in CASES)["directory_sized"]
    e = tar_entry(data, swco_tar.walk(data)[5][0])
    assert e.data is None and e.info.size == 0 and tar_entry_info(data, swco_tar.walk(data)[5][0]).size == 100
    assert _info("tarfile_8gib_minus_1").size == (8 << 30) - 1
    assert _info("tarfile_8gib_gnu").size == 8 << 30
    assert _info("tarfile_8gib_pax").size == 8 << 30


@pytest.mark.parametrize("cid,data,fmt", T.tarfile_archives(), ids=[a[0] for a in T.tarfile_archives()])
def test_tarfile_agrees(cid, data, fmt):
    n, ist, ost, gfmt, fst, recs = swco_tar.walk(data)
    assert (ist, ost, fst, gfmt) == (0, 0, 0, fmt)
    ours = [tar_entry(data, r) for r in recs]
    with tarfile.open(fileobj=io.BytesIO(data)) as t:
        members = t.getmembers()
        assert [e.info.name for e in ours] == [m.name if not m.isdir() else m.name + "/" for m in members]
        for e, m in zip(ours, members):
            assert e.info.linkName == m.linkname
            assert e.info.modificationTime == float(m.mtime) and e.info.permissions == m.mode
            if m.isdir():
                assert e.data is None
            else:
                assert e.info.size == m.size
                assert e.data == (t.extractfile(m).read() if m.isreg() else b"")
    if cid == "tarfile_pax_global":
        assert all(e.info.comment == "shared" and e.info.unknownExtendedHeaderRecords == {"vendor.key": "v"} for e in ours)


DOUBLES = [("1", 1.0), ("-1.5", -1.5), ("+2e3", 2000.0), (".5", 0.5), ("5.", 5.0), ("1e", None), ("", None), (" 1", None),
           ("1 ", None), ("\t1", None), ("0x1p4", 16.0), ("-0X.8", -0.5), ("0x", None), ("inf", math.inf), ("-Infinity", -math.inf),
           ("infi", None), ("1e400", None), ("-1e400", None), ("1e-400", None), ("0e-400", 0.0), ("4e-320", 4e-320),
           ("1_0", None), ("1\x002", 1.0), ("\x001", None), ("١", None), ("1.5e+2", 150.0), ("0x1p-1080", None)]


@pytest.mark.parametrize("text,want", DOUBLES, ids=[repr(d[0]) for d in DOUBLES])
def test_swift_double(text, want):
    assert swift_double(text) == want


def test_swift_double_nan():
    for t in ("nan", "NaN", "-nan", "nan(123)", "nan()"):
        assert math.isnan(swift_double(t))
    assert swift_double("nan(") is None
