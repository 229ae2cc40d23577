"""Hand-built ZIP containers and what ZipContainer.open / info make of them, derived from the construction and the Swift
source (Sources/ZIP/*.swift; line numbers cited per case).  Payloads come from the project's writers: deflate_writer,
bzip2_writer (and libbz2 for plain multi-block streams), lzma_writer, whose decoder model (`decode_lzma`) gives each LZMA
entry's status, output and consumed bytes — realCompSize is 9 + consumed (ZipContainer.swift:88-93).

case(shift) builds every container with `shift` bytes in front of it, so the same catalogue can be replayed with the entry
data at every residue mod 16.  A case: name, family, blob, status and entries of open(), status and entries of info(),
`engine` (the engine's documented answer where it differs from the reference, DESIGN §6), tags (what it exercises) and the
writer's Built record (extra-field steps, data offsets)."""
import bz2
import struct
import zlib

import deflate_writer as DW
import lzma_writer as LW
from bzip2_writer import Block, BZip2Writer
from zip_writer import X, Entry, build, descriptor, local_header

OK, TRAP, UNSUPPORTED = 0, 2, 6
NO_END, SIGNATURE, SIZE, VERSION, VOLUMES, ENCRYPTION, PATCHING, METHOD, LOCAL_HDR, CRC, TEXT = range(901, 912)
DEFLATE_BLOCK_TYPE, LZMA_PROPERTIES = 102, 301
WALK = {NO_END, SIGNATURE, VERSION, VOLUMES, ENCRYPTION, PATCHING, LOCAL_HDR, TEXT}   # thrown by infoWithHelper
FILLER = 0xCAFE                                                                    # an ID without a built-in reader


class Case:
    def __init__(self, name, family, built, status, wants=None, info=None, upto=None, engine=None, tags=()):
        self.name, self.family, self.built, self.blob, self.status = name, family, built, built.blob, status
        if not wants and built.cd_entries and status != OK:
            wants = [want(e) for e in built.cd_entries]      # what info() lists; open() returns nothing on a thrown error
        if info is None:
            assert status != TRAP, name                 # a trap can come from the walk or from the data: say which
            info = status if status in WALK else OK
        self.info_status = info
        if status == CRC:
            wants_all = [want(e) for e in built.cd_entries]
        else:
            wants_all = wants
        self.info_entries = [dict(w, data=None) for w in wants_all] if info == OK else []
        self.entries = wants if status == OK else wants[:upto] if status == CRC else []
        assert status != CRC or upto, name
        self.engine, self.tags = engine, set(tags)


def want(e, data=None, **over):
    """the entry as open() reports it: name from the directory, crc / size from the directory with a data descriptor and
    from the local header otherwise (ZipEntryInfo.swift:157, :184), method from the local header (:181)"""
    dd = e.lf["flags"] & 8
    w = dict(name=e.name, data=None if e.directory else (e.data if data is None else data),
             crc=(e.cf if dd else e.lf)["crc"] & 0xFFFFFFFF, size=(e.cf if dd else e.lf)["uncomp"], method=e.lf["method"],
             is_directory=e.directory, utf8=bool(e.cf["flags"] & 0x800))
    w.update(over)
    return w


def text(n, seed=0):
    words = [b"zip", b"entry", b"central", b"local", b"header", b"deflate", b"lzma", b"bzip2", b"record", b"field"]
    out, k = bytearray(), seed
    while len(out) < n:
        k = (k * 1103515245 + 12345) & 0x7FFFFFFF
        out += words[k % len(words)] + (b"\n" if k % 7 == 0 else b" ")
    return bytes(out[:n])


def deflate(data, kind="fixed"):
    """-> (payload, bit count, output)"""
    w = DW.DeflateWriter()
    if kind == "stored":
        w.stored(data, final=True)
    elif kind == "dynamic":
        w.dynamic([data] if data else [], final=True)
    else:
        w.fixed([data] if data else [], final=True)
    p, bits = w.finish()
    return p, bits, bytes(w.out)


def lzma(ops, lc=3, lp=0, pb=2, dict_size=1 << 16, usize=None, props_size=5, prop=None):
    """-> (payload, Result of decode_lzma): the 4 skipped bytes (SDK version, properties size), the properties byte, the
    dictionary size, the range-coded stream"""
    s = LW.write_lzma(ops, lc, lp, pb, dict_size)
    pbyte = LW.props_byte(lc, lp, pb) if prop is None else prop
    p = b"\x10\x02" + struct.pack("<HB", props_size, pbyte) + struct.pack("<I", dict_size & 0xFFFFFFFF) + s
    r = LW.decode_lzma(s, lc, lp, pb, dict_size, -1 if usize is None else usize)
    return p, r


def lits(data):
    return [LW.lit(b) for b in data]


def lzma_entry(name, data, end=True, declared=None, **kw):
    ops = lits(data) + ([LW.end()] if end else [])
    usize = len(data) if declared is None else declared
    p, r = lzma(ops, usize=usize, **kw)
    e = Entry(name, r.out, p, 14, uncomp=usize, crc=zlib.crc32(r.out), comp=9 + r.consumed)
    return e, r


def case_list(shift=0):
    pad = b"\xA5" * shift
    out = []

    def B(entries, prefix=b"", **kw):
        return build(entries, prefix=pad + prefix, **kw)

    def add(name, family, built, status, wants, **kw):
        out.append(Case(name, family, built, status, wants, **kw))

    # ================================================================ 1. end records (ZipContainer.swift:137-170,
    # ZipEndOfCentralDirectory.swift:21-110)
    a = Entry("a.txt", text(300, 1))
    bp, _, bo = deflate(text(500, 2))
    b = Entry("b.txt", bo, bp, 8)
    ab = [want(a), want(b)]
    add("eocd_plain", 1, B([a, b]), OK, ab)
    add("eocd_comment_0", 1, B([a, b], comment=b""), OK, ab)
    add("eocd_comment_65535", 1, B([a, b], comment=bytes(range(256)) * 255 + b"\x00" * 255), OK, ab)
    add("eocd_empty_22_bytes", 1, B([]), OK, [])
    add("eocd_prefixed_stub", 1, B([a, b], prefix=b"MZ" + bytes(1000)), OK, ab)
    # a complete look-alike record inside the comment, nearer the end: the backward probe (:147-157) takes it; it lists
    # one entry only
    real = B([a, b], comment=bytes(40))
    fake = struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, 1, 1, 0, real.cd_off, 0)
    add("eocd_lookalike_in_comment_is_taken", 1, B([a, b], comment=b"xy" + fake + bytes(16)), OK, ab[:1], tags={"lookalike"})
    # a signature in the last 21 bytes is never probed: the probe starts at size - 22 (:146)
    add("eocd_lookalike_in_last_21_bytes_ignored", 1, B([a, b], comment=b"PK\x05\x06" + bytes(17)), OK, ab)
    # a look-alike inside an entry's data (and one in the comment behind the real record): a forward search would stop at
    # the one in the data, which lists no entries
    s = Entry("sig.bin", b"data " + struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, 0, 0, 0, 0, 0) + b" more")
    add("eocd_lookalike_in_entry_data", 1, B([s, a], comment=b"PK\x05\x06 in a comment"), OK, [want(s), want(a)],
        tags={"lookalike"})
    add("eocd_archive_extra_data_record", 1, B([a, b], archive_extra=b"archive extra body"), OK, ab)
    add("eocd_archive_extra_data_record_empty", 1, B([a, b], archive_extra=b""), OK, ab)
    # saturated fields send the reader to the Zip64 locator 40 bytes in front of the end of the fixed fields (:49-59)
    for sat in (("here", "total"), ("cd_size",), ("cd_off",), ("here", "total", "cd_size", "cd_off")):
        add("zip64_eocd_saturated_" + "_".join(sat), 1, B([a, b], zip64=True, saturate=sat), OK, ab, tags={"zip64_end"})
    add("zip64_eocd_disks_saturated", 1, B([a, b], zip64=True, saturate=("disk", "cd_disk"),
                                           locator=dict(disk=0xFFFF)), OK, ab,
        tags={"zip64_end"})
    add("zip64_eocd_saturated_without_records", 1, B([a, b], saturate=("cd_off",)), SIGNATURE, [])            # :62
    add("zip64_empty_saturated_22_bytes", 1, B([], saturate=("here", "total")), TRAP, [], info=TRAP)         # offset -20
    add("zip64_locator_signature", 1, B([a, b], zip64=True, saturate=("cd_off",), locator=dict(sig=0x07064B51)), SIGNATURE, [])
    add("zip64_locator_start_disk", 1, B([a, b], zip64=True, saturate=("cd_off",), locator=dict(disk=1)), VOLUMES, [])   # :66
    add("zip64_locator_disk_count_0", 1, B([a, b], zip64=True, saturate=("cd_off",), locator=dict(disks=0)), VOLUMES, [])  # :71
    add("zip64_locator_disk_count_2", 1, B([a, b], zip64=True, saturate=("cd_off",), locator=dict(disks=2)), VOLUMES, [])
    add("zip64_record_signature", 1, B([a, b], zip64=True, saturate=("cd_off",), z64=dict(sig=0x06064B52)), SIGNATURE, [])  # :78
    add("zip64_record_needed_64", 1, B([a, b], zip64=True, saturate=("cd_off",), z64=dict(needed=64)), VERSION, [])   # :87
    add("zip64_record_needed_0x013f", 1, B([a, b], zip64=True, saturate=("cd_off",), z64=dict(needed=0x013F)), OK, ab)
    add("zip64_record_disks_differ", 1, B([a, b], zip64=True, saturate=("cd_off",), z64=dict(cd_disk=1)), VOLUMES, [])  # :93
    add("zip64_record_counts_differ", 1, B([a, b], zip64=True, saturate=("cd_off",), z64=dict(here=1)), VOLUMES, [])   # :98
    add("zip64_record_counts_override", 1, B([a, b], zip64=True, saturate=("here", "total"), z64=dict(here=1, total=1)), OK,
        ab[:1], tags={"zip64_end"})
    add("zip64_locator_end_offset_past_end", 1, B([a, b], zip64=True, saturate=("cd_off",), locator=dict(end_off=1 << 40)),
        TRAP, [], info=TRAP)

    # ================================================================ 2. extra fields
    def quirk(id, read, declared, step, central=False):
        """a field whose reader consumes `read` (len == step) whatever `declared` says; declared bytes the reader leaves
        are re-read as field headers, so they are written as a filler field (unknown ID) that ends where declared ends"""
        assert len(read) == step
        fields = [X(id, read, size=declared, step=step)]
        if declared > step:
            assert declared - step >= 4
            fields.append(X(FILLER, b"\xEE" * (declared - step - 4)))
        return fields, 4 + declared

    payload_d, _, data_d = deflate(text(900, 7), "dynamic")

    def with_local(name, fields, ext_len, family=2, status=OK, **kw):
        e = Entry(name, data_d, payload_d, 8, lextra=fields, local=dict(extra_len=ext_len))
        tail = Entry("next.txt", text(64, 3))
        add(name, family, B([e, tail]), status, [want(e), want(tail)], tags={"local_extra"}, **kw)

    def with_central(name, fields, ext_len, family=2, status=OK, **kw):
        e = Entry(name, data_d, payload_d, 8, cextra=fields, central=dict(extra_len=ext_len), comment=b"c1")
        tail = Entry("next.txt", text(64, 3), comment=b"c2")
        add(name, family, B([e, tail]), status, [want(e), want(tail)], tags={"central_extra"}, **kw)

    ntfs1 = lambda: b"\0\0\0\0" + struct.pack("<HH", 1, 24) + bytes(range(24))
    ntfs2 = lambda: b"\0\0\0\0" + struct.pack("<HH", 2, 24)
    for declared in (8, 32, 36):                        # NTFS: 4 reserved, tag, size, and 24 bytes of times only for tag 1
        for where, fn in (("local", with_local), ("central", with_central)):
            f, n = quirk(0x000A, ntfs1(), declared, 32)
            fn(f"ntfs_tag1_declared_{declared}_{where}", f, n)
            f, n = quirk(0x000A, ntfs2(), declared, 8)
            fn(f"ntfs_tag2_declared_{declared}_{where}", f, n)
    for declared in (0, 8):                             # Info-ZIP Unix: 4 bytes in a local header, the declared size in
        f, n = quirk(0x7855, b"\x01\x02\x03\x04", declared, 4)                  # the directory (BuiltinExtraFields:84-94,
        with_local(f"unix_7855_declared_{declared}_local", f, n)                # ZipCentralDirectoryEntry.swift:110)
        with_central(f"unix_7855_declared_{declared}_central", [X(0x7855, bytes(declared))], 4 + declared)
    for us in (0, 4, 8, 9):                             # new Unix: version, uid size, uid, gid size, gid; > 8 skipped
        for gs in (0, 4, 8, 9):
            body = b"\x01" + bytes([us]) + bytes(range(1, us + 1)) + bytes([gs]) + bytes(range(1, gs + 1))
            for where, fn in (("local", with_local), ("central", with_central)):
                f, n = quirk(0x7875, body, 11, len(body)) if len(body) <= 7 else ([X(0x7875, body, step=len(body))], 4 + len(body))
                fn(f"unix_7875_uid{us}_gid{gs}_{where}", f, n)
    for where, fn in (("local", with_local), ("central", with_central)):
        f, n = quirk(0x7875, b"\x02", 11, 1)            # version != 1: the reader stops after the version byte (:111)
        fn(f"unix_7875_version_2_{where}", f, n)
    # extended timestamp: the reader returns to start + size whatever the flags say (:20, :43)
    for flags, declared in ((7, 5), (1, 13), (0, 9), (7, 0)):
        body = bytes([flags]) + bytes(range(12))
        with_local(f"timestamp_flags{flags}_declared_{declared}_local", [X(0x5455, body[:declared], step=declared)], 4 + declared)
        with_central(f"timestamp_flags{flags}_declared_{declared}_central", [X(0x5455, body[:declared], step=declared)], 4 + declared)
    for id in (0x0017, 0x9901, 0xFFFF):
        with_local(f"unknown_{id:04x}_local", [X(id, b"unknown!")], 12)
        with_central(f"unknown_{id:04x}_central", [X(id, b"unknown!")], 12)
    # the last field runs past extra_len: the reader finishes it (the loop condition is checked between fields, :69)
    with_local("last_field_past_extra_len_local", [X(FILLER, bytes(20))], 10)
    with_central("last_field_past_extra_len_central", [X(FILLER, bytes(20))], 10)
    # extra_len ends inside a field header: the reader still reads the whole header and skips the declared size
    with_local("extra_len_inside_header_local", [X(FILLER, b"abc")], 2)
    with_central("extra_len_inside_header_central", [X(FILLER, b"abc")], 2)
    # two quirks in a row
    f1, n1 = quirk(0x000A, ntfs2(), 32, 8)
    f2, n2 = quirk(0x7855, b"\x01\x02\x03\x04", 8, 4)
    with_local("ntfs_then_unix_local", f1 + f2, n1 + n2)

    # the local Zip64 field: 16 bytes (uncompressed, compressed) whatever its declared size (ZipLocalHeader.swift:74-80)
    for declared in (0, 8, 16, 28):
        body = struct.pack("<QQ", len(data_d), len(payload_d))
        f, n = quirk(0x0001, body, declared, 16) if declared != 8 else ([X(0x0001, body, size=8, step=16)], 12)
        e = Entry(f"zip64_local_declared_{declared}", data_d, payload_d, 8, lextra=f,
                  local=dict(extra_len=n, comp=0xFFFFFFFF, uncomp=0xFFFFFFFF))
        tail = Entry("next.txt", text(64, 3))
        add(e.name.decode(), 2, B([e, tail]), OK, [want(e, size=len(data_d)), want(tail)], tags={"local_extra", "zip64_local"})
    # the central Zip64 field: only the saturated fields, in the order uncompressed, compressed, offset, disk (:88-101);
    # declared 28 throughout, the rest of the declared bytes is a filler field
    for mask in range(16):
        e = Entry(f"zip64_central_{mask:04b}", data_d, payload_d, 8, comment=b"after the extras")
        tail = Entry("next.txt", text(64, 3))
        built0 = B([e, tail])
        vals, cen = b"", {}
        for bit, key, v, w in ((1, "uncomp", len(data_d), "Q"), (2, "comp", len(payload_d), "Q"),
                               (4, "local_off", built0.local_off[0], "Q"), (8, "disk", 0, "I")):
            if mask & bit:
                vals += struct.pack("<" + w, v)
                cen[key] = 0xFFFF if key == "disk" else 0xFFFFFFFF
        f, n = quirk(0x0001, vals, 28, len(vals)) if len(vals) <= 24 else ([X(0x0001, vals, step=28)], 32)
        e = Entry(e.name, data_d, payload_d, 8, comment=b"after the extras", cextra=f, central=dict(cen, extra_len=n))
        add(e.name.decode(), 2, B([e, tail]), OK, [want(e), want(tail)], tags={"central_extra", "zip64_central"})

    # ================================================================ 3. text fields (LittleEndianByteReader+Zip.swift:11-98)
    names = [  # (label, bytes, utf8 flag, status)
        ("ascii", b"plain.txt", 0, OK), ("bom", b"\xEF\xBB\xBFbom.txt", 0, OK),
        ("two_byte", "café.txt".encode(), 0, OK), ("three_byte", "€.txt".encode(), 0, OK),
        ("four_byte", "\U0001F600.txt".encode(), 0, OK), ("cp437_lone_continuation", b"na\x80me", 0, OK),
        ("cp437_c0", b"\xC0\x80.txt", 0, OK), ("cp437_surrogate", b"\xED\xA0\x80", 0, OK),
        ("cp437_above_10ffff", b"\xF4\x90\x80\x80", 0, OK), ("cp437_cut_at_end", b"abc\xE2\x82", 0, OK),
        ("cp437_overlong_3", b"\xE0\x80\x80", 0, OK),
        ("needs_utf8_then_invalid", "é".encode() + b"\xFF", 0, TEXT),
        ("flag_valid", "über/\U0001F600".encode(), 0x800, OK), ("flag_ascii", b"ascii", 0x800, OK),
        ("flag_surrogate", b"\xED\xA0\x80", 0x800, TEXT), ("flag_overlong_2", b"\xC0\x80", 0x800, TEXT),
        ("flag_overlong_3", b"\xE0\x80\x80", 0x800, TEXT), ("flag_overlong_4", b"\xF0\x80\x80\x80", 0x800, TEXT),
        ("flag_above_10ffff", b"\xF4\x90\x80\x80", 0x800, TEXT), ("flag_cut_at_end", b"a\xE2\x82", 0x800, TEXT),
        ("flag_cp437_byte", b"\x80", 0x800, TEXT),
    ]
    for label, nm, flag, st in names:
        e = Entry(nm, b"named", flags=flag)
        add(f"name_{label}", 3, B([e]), st, [want(e)])
        e = Entry(b"entry", b"commented", flags=flag, comment=nm)
        add(f"comment_{label}", 3, B([e]), st, [want(e)])
        e = Entry(b"entry", b"local name", flags=flag, local_name=nm)
        add(f"local_name_{label}", 3, B([e]), st, [want(e)])

    # ================================================================ 4. entry type (ZipEntryInfo.swift:163-176)
    ents = []
    for nib in range(16):
        for dos in (0, 0x10):
            is_dir = nib == 4 or (nib not in (1, 2, 4, 6, 8, 10, 12) and dos != 0)
            ents.append(Entry(f"t{nib:x}_{dos:02x}", b"" if is_dir else b"f%d" % nib, eattr=nib << 28 | dos, directory=is_dir))
    add("entry_types", 4, B(ents), OK, [want(e) for e in ents], tags={"directory"})
    d = Entry("dir/", b"", b"directory bytes are never read", eattr=0x10, uncomp=12345, comp=5, directory=True)
    add("directory_with_size", 4, B([d, a]), OK, [want(d), want(a)], tags={"directory"})

    # ================================================================ 5. data descriptors (ZipContainer.swift:95-111)
    def dd_entry(name, data, payload, method, sig=True, wide=False, lz64=False, cz64=False, dcrc=None, dcomp=None,
                 duncomp=None, central=None):
        crc = zlib.crc32(data)
        dsc = descriptor(crc if dcrc is None else dcrc, len(payload) if dcomp is None else dcomp,
                         len(data) if duncomp is None else duncomp, sig, wide)
        lx = [X(0x0001, bytes(16))] if lz64 else []
        cx = [X(0x0001, struct.pack("<QQ", len(data), len(payload)))] if cz64 else []
        cen = dict(central or {})
        if cz64:
            cen.update(comp=0xFFFFFFFF, uncomp=0xFFFFFFFF)
        return Entry(name, data, payload, method, flags=8, local=dict(crc=0, comp=0, uncomp=0), lextra=lx, cextra=cx,
                     after=dsc, central=cen)

    dd_tail = Entry("tail.txt", text(80, 9))
    for sig in (True, False):
        for lz64 in (False, True):
            for cz64 in (False, True):
                e = dd_entry(f"dd_sig{int(sig)}_local64_{int(lz64)}_central64_{int(cz64)}", data_d, payload_d, 8, sig, lz64, lz64, cz64)
                add(e.name.decode(), 5, B([e, dd_tail]), OK, [want(e, size=len(data_d)), want(dd_tail)],
                    tags={"descriptor", "wide" if lz64 else "narrow"})
    # the central Zip64 field alone does not widen the descriptor; a wide descriptor without the local field is misread
    e = dd_entry("dd_wide_without_local64", data_d, payload_d, 8, wide=True)
    add("dd_wide_without_local64", 5, B([e, dd_tail]), SIZE, [], tags={"descriptor"})
    e = dd_entry("dd_narrow_with_local64", data_d, payload_d, 8, lz64=True)
    add("dd_narrow_with_local64", 5, B([e, dd_tail]), SIZE, [], tags={"descriptor"})
    e = dd_entry("dd_crc_differs", data_d, payload_d, 8, dcrc=1)
    add("dd_crc_differs", 5, B([e, dd_tail]), CRC, [want(e)], upto=1, tags={"descriptor"})
    e = dd_entry("dd_comp_differs", data_d, payload_d, 8, dcomp=len(payload_d) + 1)
    add("dd_comp_differs", 5, B([e, dd_tail]), SIZE, [], tags={"descriptor"})
    e = dd_entry("dd_uncomp_differs", data_d, payload_d, 8, duncomp=len(data_d) - 1)
    add("dd_uncomp_differs", 5, B([e, dd_tail]), SIZE, [], tags={"descriptor"})
    # the directory's sizes are the capacity; the descriptor's are checked: a directory size below the output still opens
    e = dd_entry("dd_central_uncomp_small", data_d, payload_d, 8, central=dict(uncomp=10))
    add("dd_central_uncomp_small", 5, B([e, dd_tail]), OK, [want(e), want(dd_tail)], tags={"descriptor", "second_decode"})
    st = dd_entry("dd_stored", b"stored with a descriptor", b"stored with a descriptor", 0)
    add("dd_stored", 5, B([st, dd_tail]), OK, [want(st), want(dd_tail)], tags={"descriptor"})
    bzp = bz2.compress(text(3000, 4), 1)
    e = dd_entry("dd_bzip2", text(3000, 4), bzp, 12, sig=False)
    add("dd_bzip2", 5, B([e, dd_tail]), OK, [want(e), want(dd_tail)], tags={"descriptor"})
    le, lr = lzma_entry("x", text(400, 5))
    e = dd_entry("dd_lzma", lr.out, le.payload, 14, lz64=True, wide=True)
    add("dd_lzma", 5, B([e, dd_tail]), OK, [want(e), want(dd_tail)], tags={"descriptor"})

    # entries whose local header sits in the archive comment, at the very end of the container
    def at_end(e, extra=b""):
        e.inline = False
        probe = B([a, e], comment=local_header(e) + e.payload + extra)
        e.cf["local_off"] = probe.eocd_off + 22
        return B([a, e], comment=local_header(e) + e.payload + extra), e

    g = Entry("g", b"stored", flags=8)
    blt, g2 = at_end(g, b"\x50\x4B\x07\x08\0\0")          # the descriptor runs past the end: a precondition failure
    add("dd_past_container_end", 5, blt, TRAP, [], info=OK)

    # ================================================================ 6. methods
    # Deflate (ZipContainer.swift:72-78)
    for kind in ("fixed", "dynamic", "stored"):
        p, bits, o = deflate(text(1000, 11), kind)
        e = Entry(f"deflate_{kind}", o, p, 8)
        add(f"deflate_{kind}", 6, B([e, a]), OK, [want(e), want(a)], tags={"mid_byte"} if bits % 8 else set())
    p, bits, o = deflate(text(1000, 11))
    # the reader is not bounded by compSize: a stream longer than it is decoded to its end, then the sizes disagree
    e = Entry("deflate_comp_short", o, p, 8, comp=len(p) - 1)
    add("deflate_stream_longer_than_comp", 6, B([e, a]), SIZE, [])
    e = Entry("deflate_comp_long", o, p + b"\0\0\0", 8, comp=len(p) + 3)
    add("deflate_stream_shorter_than_comp", 6, B([e, a]), SIZE, [])
    for more in (1, 16, 17, 4000):
        big = text(5000, 12)
        p, _, o = deflate(big, "dynamic")
        e = Entry(f"deflate_longer_by_{more}", o, p, 8, uncomp=len(o) - more)
        add(f"deflate_output_longer_than_declared_by_{more}", 6, B([e, a]), SIZE, [], tags={"second_decode"} if more > 16 else set())
    e = Entry("deflate_bad_block", b"", b"\x07", 8)
    add("deflate_wrong_block_type", 6, B([e, a]), DEFLATE_BLOCK_TYPE, [])
    # BZip2 (:79-86)
    mb = text(250000, 13)
    e = Entry("bzip2_multi_block", mb, bz2.compress(mb, 1), 12)
    add("bzip2_multi_block", 6, B([e, a]), OK, [want(e), want(a)])
    s1, s2 = bz2.compress(b"first stream", 1), bz2.compress(b"second stream", 1)
    e = Entry("bzip2_two_streams", b"first stream", s1 + s2, 12)
    add("bzip2_second_stream_inside_comp", 6, B([e, a]), SIZE, [])          # one stream is read: realCompSize = len(s1)
    w = BZip2Writer(1)
    full = [2, 2, 3, 3, 2]
    w.block(Block(symbols=[2, 3, 0, 4], used=[5, 6, 7], tables=[full, [1] * 5], selectors=[0]))
    ob, _ = w.finish()
    e = Entry("bzip2_oversubscribed", w.output(), ob, 12)
    # the reference decodes; the engine refuses an over-subscribed set even in a table no selector uses (DESIGN §6)
    add("bzip2_oversubscribed_unused_table", 6, B([e, a]), OK, [want(e), want(a)], engine=UNSUPPORTED,
        tags={"second_decode"})
    e = Entry("bzip2_longer", mb[:20000], bz2.compress(mb[:20000], 1), 12, uncomp=19990)
    add("bzip2_output_longer_than_declared", 6, B([e, a]), SIZE, [], tags={"second_decode"})
    # LZMA (:87-89, LZMAProperties.swift:49-58)
    for lc, lp, pb in ((0, 0, 0), (3, 0, 2), (0, 4, 0), (4, 0, 4), (5, 0, 0), (4, 1, 2), (3, 3, 1), (1, 4, 0), (6, 2, 3),
                       (8, 0, 1), (7, 4, 2), (8, 4, 4)):
        e, r = lzma_entry(f"lzma_lc{lc}_lp{lp}_pb{pb}", text(700, lc * 25 + lp * 5 + pb), lc=lc, lp=lp, pb=pb)
        assert r.status == OK
        add(f"lzma_lc{lc}_lp{lp}_pb{pb}", 6, B([e, a]), OK, [want(e), want(a)],
            tags={"lzma_wide", "second_decode"} if lc + lp > 4 else {"lzma"})
    for prop in (225, 255):
        e, _ = lzma_entry("p", b"x", prop=prop)
        add(f"lzma_props_{prop}", 6, B([e, a]), LZMA_PROPERTIES, [])
    for ds in (0, 1, 4095, 4096, (1 << 32) - 1):
        ops = [LW.lit(0x61), LW.match(5, 0)] + lits(b"tail") + [LW.end()]
        p, r = lzma(ops, dict_size=ds, usize=10)
        e = Entry(f"lzma_dict_{ds}", r.out, p, 14, comp=9 + r.consumed, uncomp=10)
        add(f"lzma_dict_{ds}", 6, B([e, a]), r.status, [want(e), want(a)] if r.status == OK else [], tags={"lzma"})
    for label, end, declared in (("end_marker", True, None), ("no_end_marker", False, None),
                                 ("continues_past_declared", False, 300), ("end_marker_after_declared", True, 300)):
        e, r = lzma_entry(f"lzma_{label}", text(400, 21), end=end, declared=declared)
        add(f"lzma_{label}", 6, B([e, a]), r.status, [want(e), want(a)] if r.status == OK else [], tags={"lzma"})
    for ps in (0, 7):
        e, r = lzma_entry(f"lzma_props_size_{ps}", text(200, 22), props_size=ps)
        add(f"lzma_props_size_field_{ps}", 6, B([e, a]), OK, [want(e), want(a)], tags={"lzma"})
    e, r = lzma_entry("lzma_comp_off_by_4", text(200, 23))
    e.lf["comp"] += 4
    e.cf["comp"] += 4
    add("lzma_comp_is_consumed_plus_9", 6, B([e, a]), SIZE, [])
    lz = Entry("lz", b"", b"\x10\x02\x05\x00\x5d", 14)
    blt, _ = at_end(lz)
    add("lzma_fewer_than_9_bytes_left", 6, blt, TRAP, [], info=OK)
    # stored
    z = Entry("stored_empty", b"")
    add("stored_size_0", 6, B([z, a]), OK, [want(z), want(a)])
    big = Entry("stored_past_end", b"", b"", 0, uncomp=1 << 20, comp=1 << 20, crc=0)
    add("stored_size_past_container_end", 6, B([big]), TRAP, [], info=OK)
    for m in (1, 6, 9, 93, 98, 99):
        e = Entry(f"method_{m}", b"?", b"?", m)
        add(f"method_{m}_unsupported", 6, B([a, e]), METHOD, [])
    # empty entries of every method
    ed, _, _ = deflate(b"")
    el, rl = lzma_entry("lzma_empty", b"")
    empties = [Entry("e_stored", b""), Entry("e_deflate", b"", ed, 8), Entry("e_bzip2", b"", bz2.compress(b""), 12), el]
    add("empty_entries_every_method", 6, B(empties + [a]), OK, [want(e) for e in empties] + [want(a)])

    # ================================================================ 7. order (ZipContainer.swift:47-57)
    bad = Entry("bad_deflate", b"", b"\x07", 8)
    m99 = Entry("method_99", b"?", b"?", 99)
    add("order_decode_error_before_method_error", 7, B([a, bad, m99]), DEFLATE_BLOCK_TYPE, [])
    add("order_method_error_before_decode_error", 7, B([a, m99, bad]), METHOD, [])
    p7 = Entry("props_255", b"", b"\x10\x02\x05\x00\xFF\0\0\1\0" + bytes(8), 14)
    add("order_properties_error_after_decode_error", 7, B([bad, p7]), DEFLATE_BLOCK_TYPE, [])
    add("order_properties_error_before_decode_error", 7, B([p7, bad]), LZMA_PROPERTIES, [])
    c2 = Entry("crc_bad", text(300, 30), crc=0x12345678)
    add("order_crc_then_method_error", 7, B([a, c2, m99]), CRC, [want(a), want(c2)], upto=2, tags={"crc"})
    add("order_crc_then_decode_error", 7, B([a, c2, bad]), CRC, [want(a), want(c2)], upto=2, tags={"crc"})
    add("order_decode_error_then_crc", 7, B([a, bad, c2]), DEFLATE_BLOCK_TYPE, [])
    wl, _ = lzma_entry("wide_crc_bad", text(600, 31), lc=4, lp=2, pb=1)
    wl.lf["crc"] ^= 1
    wl.cf["crc"] ^= 1
    add("order_crc_on_second_decode_then_failures", 7, B([a, wl, bad, m99]), CRC, [want(a), want(wl)], upto=2,
        tags={"crc", "second_decode"})
    add("order_crc_first_of_many", 7, B([c2, a, b]), CRC, [want(c2)], upto=1, tags={"crc"})
    add("order_directory_reversed", 7, B([a, b, c2.__class__("c.txt", b"ccc")], cd_order=[2, 1, 0]), OK,
        [want(Entry("c.txt", b"ccc")), want(b), want(a)])
    add("order_shared_local_header", 7, B([a, b], cd_order=[0, 1, 0, 0]), OK, [want(a), want(b), want(a), want(a)])
    # overlapping data: entry `inner`'s local header and data lie inside entry `outer`'s stored data
    inner = Entry("inner", b"inner data")
    blob_inner = local_header(inner) + inner.payload
    outer = Entry("outer", b"<" + blob_inner + b">")
    probe = B([outer])
    inner2 = Entry("inner", b"inner data", central=dict(local_off=probe.data_off[0] + 1), inline=False)
    add("order_overlapping_entries", 7, B([outer, inner2]), OK, [want(outer), want(inner2)])
    return out


def cases(shift=0):
    return case_list(shift)
