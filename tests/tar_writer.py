"""Hand-built TAR archives, field by field (test infrastructure): any bytes in any field, both checksum forms, base-256
and signed octal numbers, PAX records with hand-set lengths, GNU long names, any padding."""

USTAR = b"ustar\x0000"       # ustar: TarHeader.swift:101 (0x3030007261747375)
USTAR_SP = b"ustar 00"       # ustar with a space (0x3030207261747375)
GNU = b"ustar  \x00"         # GNU (0x0020207261747375)
EOF_MARKER = b"\0" * 1024


def octal(v, width):
    """`width` bytes: the octal digits, NUL-terminated, zero-padded on the left"""
    s = b"%o" % v if v >= 0 else b"-%o" % -v
    return s.rjust(width - 1, b"0") + b"\0"


def base256(v, width):
    """base-256 field (top bit set; negative values in two's complement over the field)"""
    raw = (v % (1 << (8 * width))).to_bytes(width, "big")
    return bytes([raw[0] | 0x80]) + raw[1:]


def field(v, width):
    if v is None:
        return b"\0" * width
    if isinstance(v, int):
        return octal(v, width)
    v = bytes(v)
    assert len(v) <= width, (v, width)
    return v.ljust(width, b"\0")


def header(name=b"file", mode=0o644, uid=1000, gid=1000, size=0, mtime=1700000000, chksum=None, typeflag=b"0",
           linkname=b"", magic=USTAR, uname=b"user", gname=b"group", devmajor=0, devminor=0, prefix=b"", tail=None,
           signed=False):
    """one 512-byte header.  Each numeric field takes an int (octal), bytes (written as given) or None (NULs); `tail`
    replaces bytes 345..511 (prefix / GNU times); `chksum` bytes are written as given, else the unsigned (or with `signed`,
    the signed) sum as "%06o\\0 "."""
    h = bytearray(512)
    h[0:100] = field(name, 100)
    h[100:108] = field(mode, 8)
    h[108:116] = field(uid, 8)
    h[116:124] = field(gid, 8)
    h[124:136] = field(size, 12)
    h[136:148] = field(mtime, 12)
    h[148:156] = b" " * 8
    h[156:157] = typeflag
    h[157:257] = field(linkname, 100)
    h[257:265] = field(magic, 8)
    h[265:297] = field(uname, 32)
    h[297:329] = field(gname, 32)
    h[329:337] = field(devmajor, 8)
    h[337:345] = field(devminor, 8)
    h[345:500] = field(prefix, 155)
    if tail is not None:
        h[345:345 + len(tail)] = tail
    if chksum is None:
        total = sum((b - 256 if b >= 128 else b) for b in h) if signed else sum(h)
        chksum = (b"%06o" % total if total >= 0 else b"-%05o" % -total) + b"\0 "
    h[148:156] = field(chksum, 8)
    return bytes(h)


def pad(data):
    return bytes(data) + b"\0" * (-len(data) % 512)


def entry(data=b"", **hdr):
    """a header (size defaults to len(data)) followed by its data padded to 512 bytes"""
    hdr.setdefault("size", len(data))
    return header(**hdr) + pad(data)


def record(key, value, length=None):
    """one PAX record `len key=value\\n`; `length` (int or bytes) overrides the correct length"""
    key, value = bytes(key), bytes(value)
    if length is None:
        body = b" " + key + b"=" + value + b"\n"
        n = len(body) + 1
        while len(str(n)) + len(body) != n:
            n += 1
        length = n
    if isinstance(length, int):
        length = str(length).encode()
    return length + b" " + key + b"=" + value + b"\n"


def pax(records, typeflag=b"x", name=b"PaxHeader", **hdr):
    """an extended header entry: `records` is a list of (key, value) pairs or raw bytes"""
    payload = records if isinstance(records, (bytes, bytearray)) else b"".join(record(k, v) for k, v in records)
    return entry(payload, name=name, typeflag=typeflag, **hdr)


def long_name(name, typeflag=b"L", terminate=True):
    data = bytes(name) + (b"\0" if terminate else b"")
    return entry(data, name=b"././@LongLink", typeflag=typeflag, magic=GNU)
