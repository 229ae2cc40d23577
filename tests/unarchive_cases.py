"""A named catalogue of gzip members and zlib streams for the batched unarchive calls (swc_gzip_unarchive_batch,
swc_zlib_unarchive_batch): the golden fixtures, every hand-derived header case of test_headers_cpu.py followed by a Deflate
payload and a trailer, trailer damage (CRC-32, ISIZE, Adler-32, 0-7 trailer bytes, archives of 0-19 bytes, bytes and a second
member behind the first), the Deflate catalogue of deflate_cases.py wrapped in both formats, and Python's own gzip / zlib at
levels 0-9 with every optional gzip header field.

arc.status is the status GzipArchive.unarchive / ZlibArchive.unarchive returns, read off the Swift source
(GzipArchive.swift:38-47, 79-100, ZlibArchive.swift:25-42) and the cases' own expectations, or None where only the
reference decides (a header case whose error was running out of bytes, now followed by more bytes).  arc.payload is the
output on OK and on the payload-carrying statuses, arc.consumed the archive bytes the reference read there (None: not
stated)."""
import gzip
import random
import struct
import zlib

import helpers as H
from deflate_cases import catalogue
from test_headers_cpu import GZIP_CASES, ZLIB_CASES, fixed, with_hcrc

OK, TRAP = 0, 2
WRONG_BLOCK_TYPE = 102
GZ_MAGIC, GZ_METHOD, GZ_FLAGS, GZ_HCRC, GZ_CRC, GZ_ISIZE = 601, 602, 603, 604, 605, 606
ZL_METHOD, ZL_CINFO, ZL_FCHECK, ZL_ADLER = 701, 702, 703, 705
PAYLOAD_CARRYING = (GZ_CRC, ZL_ADLER)
STATUS = {"ok": OK, "GzipError.wrongMagic": GZ_MAGIC, "GzipError.wrongCompressionMethod": GZ_METHOD,
          "GzipError.wrongFlags": GZ_FLAGS, "GzipError.wrongHeaderCRC": GZ_HCRC, "EngineError.referenceTrap": TRAP,
          "ZlibError.wrongCompressionMethod": ZL_METHOD, "ZlibError.wrongCompressionInfo": ZL_CINFO,
          "ZlibError.wrongFcheck": ZL_FCHECK}


class Arc:
    __slots__ = ("name", "fmt", "data", "status", "payload", "consumed")

    def __init__(self, name, fmt, data, status, payload=None, consumed=None):
        self.name, self.fmt, self.data, self.status = name, fmt, bytes(data), status
        self.payload, self.consumed = payload, consumed


def gzip_trailer(raw):
    return struct.pack("<II", zlib.crc32(raw), len(raw) & 0xFFFFFFFF)


def zlib_trailer(raw):
    return struct.pack(">I", zlib.adler32(raw))


def gzip_member(raw, level=6, flags=0, name=None, comment=None, extra=None, mtime=0, os_=3):
    """one gzip member with the optional fields asked for (FEXTRA's `extra` is a list of (si1, si2, bytes))"""
    h = bytearray(fixed(flags | (0x08 if name is not None else 0) | (0x10 if comment is not None else 0)
                        | (0x04 if extra is not None else 0), mtime=mtime, os_=os_))
    if extra is not None:
        area = b"".join(bytes([a, b]) + struct.pack("<H", len(d)) + d for a, b, d in extra)
        h += struct.pack("<H", len(area)) + area
    if name is not None:
        h += name + b"\0"
    if comment is not None:
        h += comment + b"\0"
    if flags & 0x02:
        h = bytearray(with_hcrc(bytes(h)))
    return bytes(h) + H.raw_deflate(raw, level) + gzip_trailer(raw)


def zlib_stream(raw, level=6, wbits=15):
    c = zlib.compressobj(level, zlib.DEFLATED, wbits)
    return c.compress(raw) + c.flush()


def golden():
    out = [Arc(rel, "gzip", H.fixture(rel), OK, H.answer(ans), len(H.fixture(rel))) for rel, ans in H.fixtures("GZip/")]
    out.append(Arc("Zlib/test_empty.zlib", "zlib", H.fixture("Zlib/test_empty.zlib"), OK, b"", 8))
    out.append(Arc("Zlib/test.zlib", "zlib", H.fixture("Zlib/test.zlib"), WRONG_BLOCK_TYPE))
    return out


HEADER_PAYLOAD = H.textlike(300, 51)
# header cases whose error is not running out of bytes keep it with a payload behind them (test_headers_cpu.py)
_KEEPS_WITH_TAIL = ("bad magic", "fextra: xlen 3", "fextra: len > rest", "fextra: xlen 5 runs over")


def header_cases():
    out = []
    body = H.raw_deflate(HEADER_PAYLOAD)
    for name, data, status, _ in GZIP_CASES:
        if data is None:
            good = with_hcrc(fixed(0x1F, mtime=7) + b"\x05\x00" + b"AB\x01\x00z" + b"name\x00" + b"cmt\x00")
            data = good.replace(b"name", b"nbme")
        arc = data + body + gzip_trailer(HEADER_PAYLOAD)
        if status == "ok":
            out.append(Arc(f"gzip header {name}", "gzip", arc, OK, HEADER_PAYLOAD, len(arc)))
        else:
            keeps = STATUS[status] not in (GZ_MAGIC, TRAP) or name in _KEEPS_WITH_TAIL
            out.append(Arc(f"gzip header {name}", "gzip", arc, STATUS[status] if keeps else None))
    for name, data, status, _ in ZLIB_CASES:
        arc = data + body + zlib_trailer(HEADER_PAYLOAD)
        if status == "ok":
            out.append(Arc(f"zlib header {name}", "zlib", arc, OK, HEADER_PAYLOAD, len(arc)))
        else:
            keeps = name not in ("one byte", "fdict without the dictionary id")
            out.append(Arc(f"zlib header {name}", "zlib", arc, STATUS[status] if keeps else None))
    return out


def trailer_cases():
    rng = random.Random(52)
    raw, other = H.textlike(5000, 53), H.textlike(3000, 54)
    g, z = gzip_member(raw), zlib_stream(raw)
    out = [Arc("gzip whole", "gzip", g, OK, raw, len(g))]
    b = bytearray(g); b[-8] ^= 1
    out.append(Arc("gzip flipped crc", "gzip", b, GZ_CRC, raw, len(g)))
    b = bytearray(g); b[-1] ^= 0x80
    out.append(Arc("gzip flipped isize", "gzip", b, GZ_ISIZE))
    for k in range(8):
        out.append(Arc(f"gzip {k} trailer bytes", "gzip", g[:len(g) - 8 + k], GZ_MAGIC))
    g0 = gzip_member(b"")
    assert len(g0) == 20
    out.append(Arc("gzip empty member, 20 bytes", "gzip", g0, OK, b"", 20))
    for k in range(20):
        out.append(Arc(f"gzip {k} bytes", "gzip", g0[:k], GZ_MAGIC))
        out.append(Arc(f"gzip {k} random bytes", "gzip", H.random_bytes(rng, k), GZ_MAGIC))
    out.append(Arc("gzip trailing bytes", "gzip", g + b"\x00\xff" * 9, OK, raw, len(g)))
    out.append(Arc("gzip second member", "gzip", g + gzip_member(other), OK, raw, len(g)))
    out.append(Arc("zlib whole", "zlib", z, OK, raw, len(z)))
    b = bytearray(z); b[-1] ^= 1
    out.append(Arc("zlib flipped adler32", "zlib", b, ZL_ADLER, raw, len(z)))
    b = bytearray(z); b[-4] ^= 0x40
    out.append(Arc("zlib flipped adler32 high byte", "zlib", b, ZL_ADLER, raw, len(z)))
    for k in range(4):
        out.append(Arc(f"zlib {k} trailer bytes", "zlib", z[:len(z) - 4 + k], ZL_ADLER, raw, len(z) - 4))
    z0 = zlib_stream(b"")
    out.append(Arc("zlib empty", "zlib", z0, OK, b"", len(z0)))
    out.append(Arc("zlib trailing bytes", "zlib", z + b"\x00\xff" * 9, OK, raw, len(z)))
    out.append(Arc("zlib second stream", "zlib", z + zlib_stream(other), OK, raw, len(z)))
    return out


GZIP_HEAD = fixed(0)
ZLIB_HEAD = b"\x78\x9c"


def deflate_member_cases():
    """the Deflate catalogue's streams that start at bit 0, each as a gzip member and as a zlib stream"""
    out = []
    for c in catalogue():
        if c.start_bit:
            continue
        if c.expect is not None:
            s = c.data[:c.stream_bytes]
            g, z = GZIP_HEAD + s + gzip_trailer(c.expect), ZLIB_HEAD + s + zlib_trailer(c.expect)
            out.append(Arc(f"gzip deflate {c.name}", "gzip", g, OK, c.expect, len(g)))
            out.append(Arc(f"zlib deflate {c.name}", "zlib", z, OK, c.expect, len(z)))
        else:
            out.append(Arc(f"gzip deflate {c.name}", "gzip", GZIP_HEAD + c.data + gzip_trailer(b""), c.status))
            out.append(Arc(f"zlib deflate {c.name}", "zlib", ZLIB_HEAD + c.data + zlib_trailer(b""), c.status))
    return out


def differential_cases():
    """Python's gzip / zlib at levels 0-9 (zlib also at every window size), with FNAME, FCOMMENT, FEXTRA and FHCRC headers"""
    rng = random.Random(55)
    out = []
    for level in range(10):
        raw = H.textlike(20000 + 1000 * level, 560 + level) if level % 3 else H.random_bytes(rng, 3000 + level)
        g = gzip.compress(raw, level, mtime=0)
        out.append(Arc(f"python gzip level {level}", "gzip", g, OK, raw, len(g)))
        for tag, kw in (("fname", dict(name=b"file.txt")), ("fcomment", dict(comment=b"caf\xe9")),
                        ("fextra", dict(extra=[(65, 66, b"xy"), (67, 68, b"")])), ("fhcrc", dict(flags=0x02)),
                        ("all", dict(name=b"n", comment=b"c", extra=[(1, 2, b"z" * 40)], flags=0x03, mtime=1700000000))):
            a = gzip_member(raw, level, **kw)
            out.append(Arc(f"gzip level {level} {tag}", "gzip", a, OK, raw, len(a)))
        z = zlib_stream(raw, level, 9 + level % 7)
        out.append(Arc(f"python zlib level {level}", "zlib", z, OK, raw, len(z)))
    return out


def cases():
    return golden() + header_cases() + trailer_cases() + deflate_member_cases() + differential_cases()


def oracle_unarchive(oracle, fmt, data):
    """the reference's (status, output, consumed bytes) for one archive; consumed as swcgpu.h states it (0 unless the status
    is OK or payload-carrying)"""
    if fmt == "gzip":
        st, out, used = oracle.gzip_unarchive(data)
        return st, out, used if st in (OK, GZ_CRC) else 0
    st, out, _ = oracle.zlib_unarchive(data)
    if st not in (OK, ZL_ADLER):
        return st, out, 0
    hl = 6 if data[1] & 0x20 else 2
    _, _, bits = oracle.deflate_decompress(data, hl * 8)
    p = hl + (bits + 7) // 8
    return st, out, p + 4 if len(data) - p >= 4 else p
