"""A named catalogue of multi-member gzip files for the member-parallel batch (swc_gzip_multi_unarchive_batch, Batch codec
'gzip_multi'): BGZF files (bgzip's layout, with and without the 28-byte EOF member), the BC subfield first, second or alone
in FEXTRA, BSIZE values that lie (short, long, past the end), members with FNAME / FCOMMENT / FHCRC, plain concatenations of
the single members of unarchive_cases.py, signature look-alikes planted in stored blocks inside BGZF and plain members,
0-byte units, garbage tails of 1-19 and 20+ bytes, and wrongCRC / wrongISize / a Deflate error in member k of m.

case.status is what GzipArchive.multiUnarchive returns, read off the Swift source (GzipArchive.swift:52-100) and the way each
case is built; case.members the members' data on OK and wrongCRC (None: not stated).  expect() gives the reference's full
answer from the oracle; zlib_starts() the member starts Python's zlib finds in a valid file."""
import random
import struct
import zlib

import helpers as H
import unarchive_cases as U

OK, GZ_MAGIC, GZ_CRC, GZ_ISIZE = U.OK, U.GZ_MAGIC, U.GZ_CRC, U.GZ_ISIZE
BGZF_BLOCK = 65280                       # bgzip's input block
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
LOOKALIKE = b"\x1f\x8b\x08\x00" + b"\x00" * 6 + b"planted look-alike member header"


class Case:
    __slots__ = ("name", "data", "status", "members")

    def __init__(self, name, data, status, members=None):
        self.name, self.data, self.status, self.members = name, bytes(data), status, members


def bgzf_member(raw, level=6, before=(), after=(), bsize_delta=0):
    """one BGZF block: FEXTRA with the BC subfield (BSIZE = block size - 1, plus `bsize_delta`) between the subfields
    `before` and `after` ((si1, si2, bytes) each)"""
    body = H.raw_deflate(raw, level) + U.gzip_trailer(raw)
    sub = lambda a, b, d: bytes([a, b]) + struct.pack("<H", len(d)) + d
    pre = b"".join(sub(*f) for f in before)
    post = b"".join(sub(*f) for f in after)
    xlen = len(pre) + 6 + len(post)
    size = 12 + xlen + len(body)
    bsize = (size - 1 + bsize_delta) & 0xFFFF
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff" + struct.pack("<H", xlen) + pre + b"BC\x02\x00" + struct.pack("<H", bsize)
            + post + body)


def bgzf(data, block=BGZF_BLOCK, eof=True, level=6):
    """bgzip's file for `data` -> (file, member payloads)"""
    parts = [data[i:i + block] for i in range(0, len(data), block)] or [b""]
    f = b"".join(bgzf_member(p, level) for p in parts)
    return (f + BGZF_EOF, parts + [b""]) if eof else (f, parts)


def planted(n, seed):
    """text with gzip signature look-alikes every ~700 bytes: stored (level 0) blocks carry them verbatim"""
    t = bytearray(H.textlike(n, seed))
    for at in range(100, n - len(LOOKALIKE), 700):
        t[at:at + len(LOOKALIKE)] = LOOKALIKE
    return bytes(t)


def bgzf_cases():
    out = []
    big = H.textlike(300000, 61)
    f, parts = bgzf(big)
    out.append(Case("bgzf 300 kB with EOF", f, OK, parts))
    f, parts = bgzf(big, eof=False)
    out.append(Case("bgzf 300 kB without EOF", f, OK, parts))
    out.append(Case("bgzf EOF member alone", BGZF_EOF, OK, [b""]))
    small = [H.textlike(700 + 90 * k, 62 + k) for k in range(6)]
    for tag, kw in (("first", {}), ("second", dict(before=[(65, 66, b"xy")])), ("first of two", dict(after=[(1, 2, b"zz")])),
                    ("last of three", dict(before=[(1, 2, b""), (3, 4, b"abc")]))):
        f = b"".join(bgzf_member(p, **kw) for p in small)
        out.append(Case(f"bgzf BC {tag}", f, OK, small))
    for tag, delta in (("short", -5), ("long", 7), ("past the end", 40000)):
        f = b"".join(bgzf_member(p, bsize_delta=delta) for p in small)
        out.append(Case(f"bgzf BSIZE {tag}", f, OK, small))
    f = b"".join(bgzf_member(p, bsize_delta=-1 if k % 2 else 0) for k, p in enumerate(small))
    out.append(Case("bgzf BSIZE off by one in every other member", f, OK, small))
    p = [planted(5000 + 300 * k, 63 + k) for k in range(4)]
    f = b"".join(bgzf_member(x, level=0) for x in p)
    out.append(Case("bgzf look-alikes in stored blocks", f + BGZF_EOF, OK, p + [b""]))
    return out


def plain_cases():
    rng = random.Random(64)
    out = []
    singles = [a for a in U.cases() if a.fmt == "gzip" and a.status == OK and a.consumed == len(a.data)]
    for g in range(0, len(singles), 7):
        grp = singles[g:g + 7]
        out.append(Case(f"concatenation {g // 7}", b"".join(a.data for a in grp), OK, [a.payload for a in grp]))
    raws = [H.textlike(2000 + 500 * k, 65 + k) for k in range(4)]
    fields = [dict(name=b"a.txt"), dict(comment=b"caf\xe9"), dict(flags=0x02), dict(name=b"n", comment=b"c", flags=0x03)]
    out.append(Case("fname fcomment fhcrc members", b"".join(U.gzip_member(r, **kw) for r, kw in zip(raws, fields)), OK, raws))
    out.append(Case("one member", U.gzip_member(raws[0]), OK, raws[:1]))
    out.append(Case("empty members", U.gzip_member(b"") * 5, OK, [b""] * 5))
    p = [planted(6000 + 200 * k, 66 + k) for k in range(3)]
    out.append(Case("plain look-alikes in stored blocks", b"".join(U.gzip_member(x, level=0) for x in p), OK, p))
    mixed = [planted(4000, 69), raws[1], raws[2]]
    out.append(Case("look-alike in member 0 of 3", b"".join(U.gzip_member(x, level=0 if k == 0 else 6) for k, x in enumerate(mixed)),
                    OK, mixed))
    whole = b"".join(U.gzip_member(r) for r in raws)
    out.append(Case("0-byte unit", b"", OK, []))
    for k in (1, 7, 19):
        out.append(Case(f"{k}-byte garbage tail", whole + H.random_bytes(rng, k), GZ_MAGIC))
        out.append(Case(f"{k}-byte zero tail", whole + b"\x00" * k, GZ_MAGIC))
    for k in (20, 33, 300):
        out.append(Case(f"{k}-byte garbage tail", whole + b"\xff" + H.random_bytes(rng, k - 1), GZ_MAGIC))
    out.append(Case("20-byte tail with the signature", whole + b"\x1f\x8b\x08\x00" + b"\x00" * 16, None))
    return out


def damage_cases():
    out = []
    raws = [H.textlike(1500 + 400 * k, 70 + k) for k in range(5)]
    mem = [U.gzip_member(r) for r in raws]
    for k in (0, 2, 4):
        m = list(mem)
        b = bytearray(m[k]); b[-8] ^= 1; m[k] = bytes(b)
        out.append(Case(f"wrongCRC in member {k} of 5", b"".join(m), GZ_CRC, raws[:k + 1]))
        m = list(mem)
        b = bytearray(m[k]); b[-1] ^= 0x40; m[k] = bytes(b)
        out.append(Case(f"wrongISize in member {k} of 5", b"".join(m), GZ_ISIZE))
        m = list(mem)
        b = bytearray(m[k]); b[10] |= 0x06; m[k] = bytes(b)           # block type 3 in the first block header
        out.append(Case(f"Deflate error in member {k} of 5", b"".join(m), U.WRONG_BLOCK_TYPE))
    small = [H.textlike(900, 75 + k) for k in range(4)]
    bm = [bgzf_member(p) for p in small]
    b = bytearray(bm[2]); b[-8] ^= 1; bm[2] = bytes(b)
    out.append(Case("bgzf wrongCRC in member 2 of 4", b"".join(bm), GZ_CRC, small[:3]))
    return out


def cases():
    return bgzf_cases() + plain_cases() + damage_cases()


def cuts(limit=4096):
    """every byte cut of the catalogue's files under `limit` bytes: (name, data) with data a proper prefix"""
    out = []
    for c in cases():
        if 0 < len(c.data) < limit:
            out += [(f"{c.name} cut {k}", c.data[:k]) for k in range(len(c.data))]
    return out


def expect(oracle, data):
    """the reference's answer: (status, output, member ends, member starts, consumed); output, table and consumed are
    empty / 0 unless the status is OK or wrongCRC"""
    st, parts, whole = oracle.gzip_multi_unarchive(data)
    if st not in (OK, GZ_CRC):
        return st, b"", [], [], 0
    ends, starts, off, total = [], [], 0, 0
    for p in parts:
        s1, _, used = oracle.gzip_unarchive(data[off:])
        assert s1 in (OK, GZ_CRC)
        starts.append(off)
        off += used
        total += len(p)
        ends.append(total)
    return st, whole, ends, starts, off


def zlib_starts(data):
    """member starts of a valid multi-member file as Python's zlib walks it (None when zlib rejects a member)"""
    starts, off = [], 0
    while off < len(data):
        d = zlib.decompressobj(31)
        try:
            d.decompress(data[off:])
        except zlib.error:
            return None
        if not d.eof:
            return None
        starts.append(off)
        off = len(data) - len(d.unused_data)
    return starts
