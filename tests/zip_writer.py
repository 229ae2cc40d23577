"""A byte-level ZIP writer for hand-built containers (no zipfile): local headers, central-directory records, the End of
Central Directory record, the Zip64 end record and locator, the archive extra data record and data descriptors, with every
field free.  Sizes and CRCs may disagree with the payload, extra fields are (id, declared size, body) triples whose body
need not be as long as declared, and the local header and the directory record of an entry are written from separate field
sets.

Each extra field carries `step`: how many bytes after its 4-byte header the reference's reader moves over it
(BuiltinExtraFields.swift:19-127, ZipLocalHeader.swift:74-80, ZipCentralDirectoryEntry.swift:88-112), stated by the case
that writes it.  The writer records, per entry and header, the reader offset after every field computed from those steps,
next to where it actually put the entry data: a case whose steps are right has the two agree (`Built.trace`)."""
import struct
import zlib

LOCAL, CENTRAL, EOCD, Z64_END, Z64_LOC, ARCHIVE_EXTRA, DESCRIPTOR = (0x04034B50, 0x02014B50, 0x06054B50, 0x06064B50,
                                                                    0x07064B50, 0x08064B50, 0x08074B50)


class X:
    """one extra field: id, body, declared size (default len(body)), reader step (default the declared size, as for an
    ID without a built-in reader: ZipLocalHeader.swift:106, ZipCentralDirectoryEntry.swift:130)"""

    def __init__(self, id, body=b"", size=None, step=None):
        self.id, self.body = id, bytes(body)
        self.size = len(self.body) if size is None else size
        self.step = self.size if step is None else step

    def bytes(self):
        return struct.pack("<HH", self.id, self.size) + self.body


def extras_bytes(fields):
    """a list of X or raw bytes (a field header cut short, say) -> the extra area"""
    return b"".join(f.bytes() if isinstance(f, X) else bytes(f) for f in fields)


def descriptor(crc, comp, uncomp, sig=True, wide=False):
    """a data descriptor: optional PK\\x07\\x08, crc, then sizes of 4 or 8 bytes"""
    w = "Q" if wide else "I"
    return (struct.pack("<I", DESCRIPTOR) if sig else b"") + struct.pack("<I" + w + w, crc, comp, uncomp)


class Entry:
    """One entry.  data: what the entry decodes to; payload: the bytes written as its data (default: data, stored).
    Header fields default to what a well-formed writer would put (crc/sizes of data/payload); `local` and `central`
    override any field of one header: version, flags, method, time, date, crc, comp, uncomp, name_len, extra_len, plus
    made_by, comment_len, disk, iattr, eattr, local_off (central only).  lextra / cextra: the extra fields of each header.
    after: bytes written after the payload (a data descriptor, or whatever the next header is preceded by)."""

    def __init__(self, name, data=b"", payload=None, method=0, *, flags=0, time=0x6000, date=0x5264, crc=None, comp=None,
                 uncomp=None, version=20, made_by=0x031E, eattr=0, iattr=0, comment=b"", lextra=(), cextra=(),
                 after=b"", local=None, central=None, local_name=None, directory=False, inline=True):
        self.name = name.encode() if isinstance(name, str) else bytes(name)
        self.local_name = self.name if local_name is None else bytes(local_name)
        self.data = bytes(data)
        self.payload = self.data if payload is None else bytes(payload)
        self.directory = directory
        base = dict(version=version, flags=flags, method=method, time=time, date=date,
                    crc=zlib.crc32(self.data) if crc is None else crc,
                    comp=len(self.payload) if comp is None else comp, uncomp=len(self.data) if uncomp is None else uncomp)
        self.lf = dict(base, **(local or {}))
        self.cf = dict(base, made_by=made_by, disk=0, iattr=iattr, eattr=eattr)
        self.cf.update(central or {})
        self.comment = bytes(comment)
        self.lextra, self.cextra = list(lextra), list(cextra)
        self.after = bytes(after)
        self.inline = inline                 # False: no local header of its own (the record's local_off points elsewhere)


def local_header(e):
    f, ex = e.lf, extras_bytes(e.lextra)
    return struct.pack("<IHHHHHIIIHH", LOCAL, f["version"], f["flags"], f["method"], f["time"], f["date"], f["crc"] & 0xFFFFFFFF,
                       f["comp"], f["uncomp"], f.get("name_len", len(e.local_name)), f.get("extra_len", len(ex))) + e.local_name + ex


def central_record(e, local_off):
    f, ex = e.cf, extras_bytes(e.cextra)
    return struct.pack("<IHHHHHHIIIHHHHHII", CENTRAL, f["made_by"], f["version"], f["flags"], f["method"], f["time"], f["date"],
                       f["crc"] & 0xFFFFFFFF, f["comp"], f["uncomp"], f.get("name_len", len(e.name)), f.get("extra_len", len(ex)),
                       f.get("comment_len", len(e.comment)), f["disk"], f["iattr"], f["eattr"],
                       f.get("local_off", local_off)) + e.name + ex + e.comment


class Built:
    """blob: the container; local_off / data_off: per entry (list order); cd_off, eocd_off; trace: per entry and header
    {"fields": [(id, declared, step, reader offset after it)], "reader_end": where the steps put the reader after the
    extra area, "data_off": where the writer put the data (local) or the comment (central)}"""

    def __init__(self):
        self.blob, self.local_off, self.data_off, self.trace = b"", [], [], []
        self.cd_off = self.eocd_off = None


def _walk(fields, start):
    at, out = start, []
    for f in fields:
        if not isinstance(f, X):
            return None, out                        # a raw fragment: the case states its own outcome
        at += 4 + f.step
        out.append((f.id, f.size, f.step, at))
    return at, out


def build(entries, *, cd_order=None, comment=b"", prefix=b"", between=b"", archive_extra=None, eocd=None, zip64=False,
          z64=None, locator=None, saturate=(), tail=b""):
    """entries in local-header order; cd_order: entry indices in directory order (repeats allowed: records sharing a local
    header).  archive_extra: the body of an archive extra data record in front of the directory.  eocd / z64 / locator:
    field overrides of the end records (eocd: disk, cd_disk, here, total, cd_size, cd_off, comment_len; z64: sig, size,
    made_by, needed, disk, cd_disk, here, total, cd_size, cd_off; locator: sig, disk, end_off, disks).  zip64: write the
    Zip64 end record and locator; saturate: EOCD fields written as 0xFFFF / 0xFFFFFFFF.  between: bytes between the last
    entry and the directory; tail: bytes after the end record's comment."""
    b = Built()
    out = bytearray(prefix)
    for e in entries:
        if not e.inline:
            b.local_off.append(None), b.data_off.append(None), b.trace.append({})
            continue
        b.local_off.append(len(out))
        h = local_header(e)
        out += h
        b.data_off.append(len(out))
        name_end = b.local_off[-1] + 30 + len(e.local_name)
        end, fields = _walk(e.lextra, name_end)
        b.trace.append({"local": {"fields": fields, "reader_end": end, "data_off": len(out)}})
        out += e.payload + e.after
    out += between
    cd_start = len(out)
    if archive_extra is not None:
        out += struct.pack("<II", ARCHIVE_EXTRA, len(archive_extra)) + archive_extra
    order = list(range(len(entries))) if cd_order is None else list(cd_order)
    b.cd_entries = [entries[i] for i in order]
    for i in order:
        e = entries[i]
        rec_off = len(out)
        out += central_record(e, b.local_off[i] or 0)
        end, fields = _walk(e.cextra, rec_off + 46 + len(e.name))
        b.trace[i].setdefault("central", {"fields": fields, "reader_end": end,
                                          "data_off": rec_off + 46 + len(e.name) + len(extras_bytes(e.cextra))})
    cd_size = len(out) - cd_start
    n = len(order)
    if zip64:
        z = dict(sig=Z64_END, size=44, made_by=45, needed=45, disk=0, cd_disk=0, here=n, total=n, cd_size=cd_size, cd_off=cd_start)
        z.update(z64 or {})
        z64_off = len(out)
        out += struct.pack("<IQHHIIQQQQ", z["sig"], z["size"], z["made_by"], z["needed"], z["disk"], z["cd_disk"], z["here"],
                           z["total"], z["cd_size"], z["cd_off"])
        lo = dict(sig=Z64_LOC, disk=0, end_off=z64_off, disks=1)
        lo.update(locator or {})
        out += struct.pack("<IIQI", lo["sig"], lo["disk"], lo["end_off"], lo["disks"])
    f = dict(disk=0, cd_disk=0, here=n, total=n, cd_size=cd_size, cd_off=cd_start, comment_len=len(comment))
    for k in saturate:
        f[k] = 0xFFFF if k in ("disk", "cd_disk", "here", "total") else 0xFFFFFFFF
    f.update(eocd or {})
    b.eocd_off, b.cd_off = len(out), cd_start
    out += struct.pack("<IHHHHIIH", EOCD, f["disk"] & 0xFFFF, f["cd_disk"] & 0xFFFF, f["here"] & 0xFFFF, f["total"] & 0xFFFF,
                       f["cd_size"] & 0xFFFFFFFF, f["cd_off"] & 0xFFFFFFFF, f["comment_len"]) + comment + tail
    b.blob = bytes(out)
    return b
