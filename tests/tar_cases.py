"""Catalogue of TAR archives with the statuses TarContainer.info / open / formatOf give them, derived from the reference
(Sources/TAR/*.swift, cited per case).  Each case: (id, data, info status, open status, formatOf status, format, number of
entry records).  Statuses are include/swc_status.h codes; SWC_ERR_REFERENCE_TRAP (2) stands where Swift traps or never
returns."""
import io
import tarfile

import tar_writer as W

OK, TRAP = 0, 2
SMALL, FIELD, CHK, PAXE = 1001, 1002, 1003, 1004
PRE, USTAR, GNU, PAX = 0, 1, 2, 3
E = W.EOF_MARKER


def _tarfile(fmt, members, pax_headers=None):
    b = io.BytesIO()
    with tarfile.open(fileobj=b, mode="w", format=fmt, pax_headers=pax_headers) as t:
        for ti, data in members:
            t.addfile(ti, io.BytesIO(data) if data is not None else None)
    return b.getvalue()


def _ti(name, data=b"", type=tarfile.REGTYPE, linkname="", mtime=1700000000, mode=0o644):
    ti = tarfile.TarInfo(name)
    ti.type, ti.linkname, ti.mtime, ti.mode = type, linkname, mtime, mode
    ti.size = len(data) if type in (tarfile.REGTYPE,) else 0
    ti.uname, ti.gname = "user", "group"
    return ti, (data if type == tarfile.REGTYPE else None)


def tarfile_members():
    """member lists written by tarfile in every format: long and Unicode names, long link names, symlinks, directories,
    empty files"""
    long = "deep/" * 30 + "file.txt"
    return [
        ("dir", _ti("dir/", type=tarfile.DIRTYPE, mode=0o755)),
        ("file", _ti("dir/hello.txt", b"hello, world\n" * 7)),
        ("empty", _ti("dir/empty", b"")),
        ("block", _ti("dir/block.bin", bytes(range(256)) * 4)),
        ("odd", _ti("dir/odd.bin", b"\x01" * 513)),
        ("symlink", _ti("dir/link", type=tarfile.SYMTYPE, linkname="hello.txt")),
        ("hardlink", _ti("dir/hard", type=tarfile.LNKTYPE, linkname="dir/hello.txt")),
        ("long", _ti(long, b"long name\n")),
        ("longlink", _ti("dir/longlink", type=tarfile.SYMTYPE, linkname="target/" * 20 + "t")),
    ]


def tarfile_archives():
    """(id, bytes, format) where the reference and tarfile must agree on names, sizes and data"""
    out = []
    base = [m for _, m in tarfile_members()]
    uni = [_ti("grüße/日本語.txt", "ünïcödé\n".encode())]
    out.append(("tarfile_gnu", _tarfile(tarfile.GNU_FORMAT, base + uni), GNU))
    out.append(("tarfile_pax", _tarfile(tarfile.PAX_FORMAT, base + uni), PAX))
    short = [m for k, m in tarfile_members() if k not in ("long", "longlink")]
    out.append(("tarfile_ustar", _tarfile(tarfile.USTAR_FORMAT, short), USTAR))
    out.append(("tarfile_pax_global", _tarfile(tarfile.PAX_FORMAT, short, pax_headers={"comment": "shared", "vendor.key": "v"}), PAX))
    return out


def _huge(fmt, size):
    """a header-only archive whose entry claims `size` bytes (8 GiB - 1 fits octal; 8 GiB needs base-256 / PAX)"""
    ti = tarfile.TarInfo("big.bin")
    ti.size = size
    return ti.tobuf(fmt, "utf-8", "surrogateescape")


def cases():
    c = []
    add = lambda *a: c.append(a)
    f1 = W.entry(b"hello", name=b"a.txt")
    # ---- end of the walk (TarParser.swift:36-42) ----
    add("empty", b"", OK, OK, OK, PRE, 0)                                      # isFinished at once
    add("eof_only", E, OK, OK, OK, PRE, 0)
    add("one_file", f1 + E, OK, OK, OK, USTAR, 1)
    add("behind_eof_ignored", f1 + E + b"\x01" * 700, OK, OK, OK, USTAR, 1)
    add("no_eof_room_left", f1, OK, OK, OK, USTAR, 1)                         # dataEnd 517 < 1024
    add("no_eof_data_to_end", W.entry(b"x" * 512), OK, SMALL, OK, USTAR, 1)  # dataEnd == count: open :208
    add("truncated_tail", f1 + b"\x01" * 100, SMALL, SMALL, SMALL, PRE, 1)    # bytesLeft < 512 :40
    add("truncated_only", b"\x01" * 511, SMALL, SMALL, SMALL, PRE, 0)
    add("zero_block_then_data", f1 + b"\0" * 512 + b"\x01" * 512, FIELD, FIELD, FIELD, PRE, 1)
    add("zero_block_at_end", f1 + b"\0" * 512, FIELD, FIELD, FIELD, PRE, 1)
    add("zero_block_then_short", f1 + b"\0" * 1023, FIELD, FIELD, FIELD, PRE, 1)
    # ---- field order and checksum (TarHeader.swift:56-91) ----
    add("size_bad_before_checksum", W.header(size=b"abc", chksum=b"1\0") + E, FIELD, FIELD, FIELD, PRE, 0)
    add("checksum_unparsable", W.header(chksum=b"xyz\0") + E, CHK, CHK, CHK, PRE, 0)
    add("checksum_mismatch", W.header(chksum=b"000001\0 ") + E, CHK, CHK, CHK, PRE, 0)
    add("checksum_signed", W.entry(b"s", name="ü€".encode(), signed=True) + E, OK, OK, OK, USTAR, 1)
    add("checksum_unsigned_high", W.entry(b"s", name="ü€".encode()) + E, OK, OK, OK, USTAR, 1)
    add("checksum_signed_mismatch", W.entry(b"s", name="ü€".encode(), chksum=b"1\0") + E, CHK, CHK, CHK, PRE, 0)
    # ---- tarInt (LittleEndianByteReader+Tar.swift:38-91) ----
    add("octal_12_digits_lose_last", W.header(size=b"000000000012") + W.pad(b"x") + E, OK, OK, OK, USTAR, 1)
    add("octal_only_last_byte", W.header(size=b"\0" * 11 + b"5") + E, FIELD, FIELD, FIELD, PRE, 0)
    add("octal_leading_space_nul", W.header(size=b" \0 5\0", mode=b"\0" * 7 + b"7") + W.pad(b"12345") + E, OK, OK, OK, USTAR, 1)
    add("octal_signs", W.header(size=b"+1\0", uid=b"-7\0", gid=b"+0\0") + W.pad(b"z") + E, OK, OK, OK, USTAR, 1)
    add("octal_space_terminated", W.header(size=b"3 9\0", mtime=b"17 \0") + W.pad(b"abc") + E, OK, OK, OK, USTAR, 1)
    add("octal_bad_digit", W.header(uid=b"8\0", mode=b"x\0") + E, OK, OK, OK, USTAR, 1)
    add("base256_size", W.header(size=W.base256(1, 12), uid=W.base256(1 << 40, 8)) + W.pad(b"q") + E, OK, OK, OK, USTAR, 1)
    add("base256_negative", W.header(mtime=W.base256(-86400, 12), uid=W.base256(-1, 8)) + E, OK, OK, OK, USTAR, 1)
    add("base256_overflow_size", W.header(size=b"\x80\0\0\x01" + b"\0" * 8) + E, FIELD, FIELD, FIELD, PRE, 0)
    add("base256_overflow_mtime", W.header(mtime=b"\x80\x01" + b"\0" * 10) + E, OK, OK, OK, USTAR, 1)
    # ---- layout (TarHeader.swift:93-134) ----
    add("gnu_times", W.entry(b"g", magic=W.GNU, tail=W.octal(1600000000, 12) + W.octal(1500000000, 12)) + E, OK, OK, OK, GNU, 1)
    add("ustar_space_magic", W.entry(b"u", magic=W.USTAR_SP) + E, OK, OK, OK, USTAR, 1)
    add("pre_posix", W.entry(b"p", magic=b"\0" * 8, uname=b"ignored") + E, OK, OK, OK, PRE, 1)
    add("prefix", W.entry(b"p", name=b"f", prefix=b"dir") + W.entry(b"q", name=b"g", prefix=b"dir/") + E, OK, OK, OK, USTAR, 2)
    add("prefix_gnu_ignored", W.entry(b"p", name=b"f", magic=W.GNU, prefix=b"dir") + E, OK, OK, OK, GNU, 1)
    add("bad_utf8_name", W.entry(b"b", name=b"a\xffb\xc3", linkname=b"\xe2\x82") + E, OK, OK, OK, USTAR, 1)
    add("types", b"".join(W.entry(name=b"t%c" % t, typeflag=bytes([t])) for t in b"\x0001234567AS") + E, OK, OK, OK, USTAR, 11)
    add("directory_sized", W.entry(name=b"d/", typeflag=b"5", size=100), OK, OK, OK, USTAR, 1)
    # ---- special entries (TarParser.swift:51-69, TarExtendedHeader.swift:31-101) ----
    add("gnu_long_name", W.long_name(b"n" * 300) + W.entry(b"L", name=b"short") + E, OK, OK, OK, GNU, 1)
    add("gnu_long_name_unterminated", W.long_name(b"m" * 100, terminate=False) + W.entry(b"L") + E, OK, OK, OK, GNU, 1)
    add("gnu_long_link", W.long_name(b"k" * 200, b"K") + W.entry(typeflag=b"2", linkname=b"s") + E, OK, OK, OK, GNU, 1)
    add("long_name_resets", W.long_name(b"n" * 120) + W.entry(b"1") + W.entry(b"2", name=b"plain") + E, OK, OK, OK, GNU, 2)
    add("pax_local", W.pax([(b"path", "päx/name".encode()), (b"size", b"3"), (b"uid", b"4294967296"), (b"mtime", b"1700000000.5"),
                            (b"uname", b"pu"), (b"gname", b"pg"), (b"linkpath", b"lp"), (b"charset", b"ISO-IR 10646 2000 UTF-8"),
                            (b"comment", b"c"), (b"gid", b"-3"), (b"atime", b"1.25"), (b"ctime", b"-2.5e1"), (b"vendor.x", b"y")])
        + W.entry(b"hello") + E, OK, OK, OK, PAX, 1)
    add("pax_global_persists", W.pax([(b"comment", b"g1"), (b"mtime", b"5"), (b"g.k", b"1")], b"g") + W.pax([(b"path", b"l1"), (b"g.k", b"2")])
        + W.entry(b"a") + W.entry(b"b", name=b"second") + E, OK, OK, OK, PAX, 2)
    add("pax_sun_x", W.pax([(b"path", b"sun")], b"X") + W.entry(b"a") + E, OK, OK, OK, USTAR, 1)
    add("pax_sun_x_prePosix", W.pax([(b"path", b"sun")], b"X", magic=b"\0" * 8) + W.entry(b"a", magic=b"\0" * 8) + E, OK, OK, OK, PRE, 1)
    add("pax_empty", W.pax(b"") + W.entry(b"e") + E, OK, OK, OK, PAX, 1)
    add("pax_negative_length", W.pax(b"-1 k=\n") + W.entry(b"e") + E, OK, OK, OK, PAX, 1)
    add("pax_plus_length", W.pax(b"+11 k=abcd\n") + W.entry(b"e") + E, OK, OK, OK, PAX, 1)
    add("pax_bad_length", W.pax(b"1x k=v\n") + W.entry(b"e") + E, PAXE, PAXE, PAXE, PRE, 0)
    add("pax_empty_length", W.pax(b" k=v\n") + W.entry(b"e") + E, PAXE, PAXE, PAXE, PRE, 0)
    add("pax_key_not_utf8", W.pax(W.record(b"\xff", b"v")) + W.entry(b"e") + E, PAXE, PAXE, PAXE, PRE, 0)
    add("pax_value_not_utf8_skipped", W.pax([(b"path", b"good"), (b"path", b"\xff"), (b"x.k", b"\xfe")]) + W.entry(b"e") + E, OK, OK, OK, PAX, 1)
    add("pax_not_newline", W.pax(W.record(b"path", b"abc", 10)) + W.entry(b"e") + E, PAXE, PAXE, PAXE, PRE, 0)
    add("pax_scan_past_end", W.pax(b"abc") + W.entry(b"e") + E, TRAP, TRAP, TRAP, PRE, 0)
    add("pax_no_equals", W.pax(b"5 abc") + W.entry(b"e") + E, TRAP, TRAP, TRAP, PRE, 0)
    add("pax_length_past_end", W.pax(b"99 k=v\n") + W.entry(b"e") + E, TRAP, TRAP, TRAP, PRE, 0)
    add("pax_int_overwritten_nil", W.pax([(b"uid", b"5"), (b"uid", b" 6"), (b"size", b"1"), (b"size", b"x")]) + W.entry(b"e", uid=9) + E,
        OK, OK, OK, PAX, 1)
    add("pax_time_falls_through", W.pax([(b"mtime", b"12.5"), (b"atime", b"0x1p4")], b"g") + W.pax([(b"mtime", b"abc"), (b"ctime", b" 1")])
        + W.entry(b"e", magic=W.GNU, tail=W.octal(7, 12) + W.octal(8, 12)) + E, OK, OK, OK, PAX, 1)
    add("pax_value_with_newline", W.pax([(b"comment", b"two\nlines")]) + W.entry(b"e") + E, OK, OK, OK, PAX, 1)
    add("pax_size_cuts_open", W.pax([(b"size", b"3")]) + W.entry(b"hello") + E, OK, OK, OK, PAX, 1)
    add("pax_size_past_end", W.pax([(b"size", b"100000")]) + W.entry(b"hello") + E, OK, SMALL, OK, PAX, 1)
    add("pax_size_negative", W.pax([(b"size", b"-1")]) + W.entry(b"hello") + E, OK, TRAP, OK, PAX, 1)
    add("pax_size_overflow", W.pax([(b"size", b"9223372036854775807")]) + W.entry(b"hello") + E, OK, TRAP, OK, PAX, 1)
    add("pax_size_directory", W.pax([(b"size", b"-1")]) + W.entry(name=b"d/", typeflag=b"5") + E, OK, OK, OK, PAX, 1)
    # ---- traps and hangs ----
    add("special_past_end", W.header(name=b"L", typeflag=b"L", size=4096, magic=W.GNU) + W.pad(b"n"), TRAP, TRAP, TRAP, PRE, 0)
    add("special_negative", W.header(typeflag=b"x", size=b"-1\0") + E, TRAP, TRAP, TRAP, PRE, 0)
    add("round512_overflow", W.header(size=W.base256((1 << 63) - 1, 12), magic=W.GNU) + E, TRAP, TRAP, TRAP, PRE, 0)
    add("round512_overflow_special", W.header(size=W.base256((1 << 63) - 600, 12), typeflag=b"L") + E, TRAP, TRAP, TRAP, PRE, 0)
    add("cycle_self", W.header(size=b"-1000\0") + E, TRAP, TRAP, TRAP, PRE, 2 * 3 + 2)
    add("cycle_gnu_returns", W.header(size=b"-1000\0", magic=W.GNU) + E, TRAP, TRAP, OK, GNU, 2 * 3 + 2)
    add("before_start", f1 + W.header(size=b"-4000\0") + E, TRAP, TRAP, TRAP, PRE, 2)
    back = W.header(name=b"A", size=512) + W.header(name=b"B", size=512) + W.header(name=b"C", size=b"-2000\0") + E
    # A (0) skips its data block B, C (1024) steps back 1 024 bytes to B (512), B goes on to the EOF marker at 1536
    add("negative_moves_back", back, OK, TRAP, OK, USTAR, 3)
    # ---- formatOf returns early (TarContainer.swift:40-70) ----
    add("format_gnu_hides_error", W.entry(b"g", magic=W.GNU) + W.header(chksum=b"1\0") + E, CHK, CHK, OK, GNU, 1)
    add("format_pax_hides_trap", W.pax([(b"a", b"b")]) + W.entry(b"x") + W.pax(b"zz"), TRAP, TRAP, OK, PAX, 1)
    add("format_long_hides_truncation", W.long_name(b"z" * 10) + W.entry(b"x") + b"\x01" * 10, SMALL, SMALL, OK, GNU, 1)
    # ---- the reference's named test files (Tests/TarTests.swift:72-370), restated in their shapes; REFERENCE_FIELDS below
    # holds what each of those tests asserts ----
    own = dict(uid=501, gid=20, uname=b"timofeysolomko", gname=b"staff", mode=0o644)
    gnu_times = W.octal(1500000001, 12) + W.octal(1500000002, 12)
    add("test_big_num_field", W.header(name=b"rands", size=W.base256(8600000000, 12), magic=W.GNU, tail=gnu_times, **own),
        OK, SMALL, OK, GNU, 1)                                           # no data: the file is cut after its header
    add("test_negative_mtime", W.entry(b"File with negative mtime.\n\n", name=b"file", magic=W.GNU,
                                       mtime=W.base256(-313006414, 12), **own) + E, OK, OK, OK, GNU, 1)
    add("test_pax_record_newline", W.pax([(b"mtime", b"1666443016"), (b"SCHILY.note", b"weird\nvalue")])
        + W.entry(b"Hello, weird pax record value!", name=b"test_file", uid=501, gid=20, uname=b"tsolomko", gname=b"staff",
                  mode=0o644) + E, OK, OK, OK, PAX, 1)
    add("test_only_dir_header", W.header(name=b"empty_dir/", typeflag=b"5", **dict(own, mode=0o755)), OK, OK, OK, USTAR, 1)
    add("test_empty_cont", b"\0" * 10240, OK, OK, OK, PRE, 0)
    add("test_gnu_inc_format", W.entry(b"Yfile1\0Yfile2\0\0", name=b"dir/", typeflag=b"D", magic=W.GNU, tail=gnu_times, **own)
        + W.entry(b"one\n", name=b"dir/file1", magic=W.GNU, tail=gnu_times, **own)
        + W.entry(b"two\n", name=b"dir/file2", magic=W.GNU, tail=gnu_times, **own) + E, OK, OK, OK, GNU, 3)
    answer = "Текстовый файл с юникодом.\n".encode()
    add("test_unicode_pax", W.pax([(b"path", "текстовый файл.answer".encode())]) + W.entry(answer, name=b"PaxHeaders/answer", **own) + E,
        OK, OK, OK, PAX, 1)
    add("test_unicode_ustar", W.entry(answer, name="текстовый файл.answer".encode(), **own) + E, OK, OK, OK, USTAR, 1)
    # ---- tarfile ----
    for cid, data, fmt in tarfile_archives():
        add(cid, data, OK, OK, OK, fmt, None)
    add("tarfile_8gib_minus_1", _huge(tarfile.USTAR_FORMAT, (8 << 30) - 1) + E, OK, SMALL, OK, USTAR, 1)
    add("tarfile_8gib_gnu", _huge(tarfile.GNU_FORMAT, 8 << 30) + E, OK, SMALL, OK, GNU, 1)
    add("tarfile_8gib_pax", _huge(tarfile.PAX_FORMAT, 8 << 30) + E, OK, SMALL, OK, PAX, 1)
    return c


# what the reference's tests assert about each named file's entries (TarTests.swift), as TarEntryInfo fields, plus the
# entry data where they check it; "*" means "not None"
_OWNER = dict(ownerID=501, groupID=20, ownerUserName="timofeysolomko", ownerGroupName="staff")
REFERENCE_FIELDS = {
    "test_big_num_field": [dict(_OWNER, name="rands", type="regular", size=8600000000, permissions=420, comment=None)],
    "test_negative_mtime": [dict(_OWNER, name="file", type="regular", size=27, permissions=420, modificationTime=-313006414.0,
                                 comment=None, data=b"File with negative mtime.\n\n")],
    "test_pax_record_newline": [dict(name="test_file", type="regular", size=30, accessTime=None, creationTime=None,
                                     modificationTime=1666443016.0, permissions=420, ownerID=501, groupID=20,
                                     ownerUserName="tsolomko", ownerGroupName="staff", deviceMajorNumber=0,
                                     deviceMinorNumber=0, charset=None, comment=None, linkName="",
                                     data=b"Hello, weird pax record value!")],
    "test_only_dir_header": [dict(_OWNER, name="empty_dir/", type="directory", size=0, permissions=493, comment=None, data=None)],
    "test_empty_cont": [],
    "test_gnu_inc_format": [dict(_OWNER, accessTime="*", creationTime="*")] * 3,
    "test_unicode_pax": [dict(_OWNER, name="текстовый файл.answer", type="regular", permissions=420, comment=None,
                              data="Текстовый файл с юникодом.\n".encode())],
    "test_unicode_ustar": [dict(_OWNER, name="текстовый файл.answer", type="regular", permissions=420, comment=None,
                                data="Текстовый файл с юникодом.\n".encode())],
}
# the formats the reference's tests assert with formatOf
REFERENCE_FORMATS = {"test_big_num_field": GNU, "test_negative_mtime": GNU, "test_pax_record_newline": PAX,
                     "test_only_dir_header": USTAR, "test_empty_cont": PRE, "test_gnu_inc_format": GNU,
                     "test_unicode_pax": PAX, "test_unicode_ustar": USTAR}

SMALL_CUTS = ("one_file", "prefix", "gnu_long_name", "pax_local", "pax_global_persists", "negative_moves_back", "gnu_times")
