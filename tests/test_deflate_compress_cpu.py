"""The CPU restatement of Deflate.compress, GzipArchive.archive and ZlibArchive.archive (oracle/deflate_compress.c)
against streams derived by hand from the Swift source, against a plain-Python statement of the parse (whose near-miss
variants show that each catalogue edge discriminates), and through zlib, gzip and the existing oracle decoder."""
import gzip
import struct
import zlib

import pytest

import deflatec_cases as K
import helpers as H

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]


@pytest.fixture(scope="module")
def oc():
    import swco_deflatec
    swco_deflatec.lib()
    return swco_deflatec


def _lsym(length):
    s = max(i for i, b in enumerate(LEN_BASE) if b <= length)
    return 257 + s


def _dsym(distance):
    return max(i for i, b in enumerate(DIST_BASE) if b <= distance)


def statement(data, variant=None):
    """Deflate.compress(data:) in Python, line by line (Deflate+Compress.swift:22-197).  `variant` names one near miss."""
    n = len(data)
    table, codes = {}, []
    key = (lambda i: (data[i] << 16 | data[i + 1] << 8 | data[i + 2]) & 0xFFF) if variant == "bucket" else \
          (lambda i: data[i] << 16 | data[i + 1] << 8 | data[i + 2])
    i = 0
    while i < n - 2:                                                    # :143
        k = key(i)
        if k not in table:
            table[k] = i
            codes.append(data[i]); i += 1
            continue
        start = table[k]
        far = (i - start >= 32768) if variant == "lt_32768" else (i - start > 32768)
        if not (far and variant == "no_record_far"):
            table[k] = i                                                # :158
        if far:
            codes.append(data[i]); i += 1
            continue
        length = 3
        while i + length < n and data[i + length] == data[start + length] and length < 258:
            length += 1
        if variant == "record_inside":
            for p in range(i + 1, min(i + length, n - 2)):
                table[key(p)] = p
        codes.append((length, i - start))
        i += length
    codes.extend(data[i:])
    bits = 3 + 7
    for c in codes:
        if isinstance(c, int):
            bits += 8 if c < 144 else 9
        else:
            ls, ds = _lsym(c[0]), _dsym(c[1])
            bits += (7 if ls <= 279 else 8) + (0 if ls <= 260 or ls == 285 else ((ls - 257) >> 2) - 1)
            bits += 5 + (0 if ds < 2 else (ds >> 1) - 1)
    static = (bits + 7) // 8
    stored_size = n + 5
    fits = (n <= 65535) if variant == "limit_n" else (stored_size <= 65535)
    smaller = (stored_size < static) if variant == "strict_tie" else (stored_size <= static)
    if smaller and fits:
        return bytes([1, n & 0xFF, (n >> 8) & 0xFF, (n ^ 0xFFFF) & 0xFF, ((n ^ 0xFFFF) >> 8) & 0xFF]) + data
    w = H.LsbBitWriter()
    w.write_bits([1, 1, 0])

    def code(v, ln):
        w.write_bits([(v >> k) & 1 for k in range(ln - 1, -1, -1)])

    def lit(s):
        if s <= 143:
            code(0x30 + s, 8)
        elif s <= 255:
            code(0x190 + s - 144, 9)
        elif s <= 279:
            code(s - 256, 7)
        else:
            code(0xC0 + s - 280, 8)

    for c in codes:
        if isinstance(c, int):
            lit(c)
            continue
        ls, ds = _lsym(c[0]), _dsym(c[1])
        lit(ls)
        w.write_number(c[0] - LEN_BASE[ls - 257], 0 if ls <= 260 or ls == 285 else ((ls - 257) >> 2) - 1)
        code(ds, 5)
        w.write_number(c[1] - DIST_BASE[ds], 0 if ds < 2 else (ds >> 1) - 1)
    lit(256)
    w.align()
    return w.data


# hand-derived from the Swift source: header bits 1, 1, 0; fixed codes most significant bit first; EOB 0000000
HAND = {
    b"": "0300",
    b"a": "4b0400",
    b"ab": "4b4c0200",
    b"abc": "4b4c4a0600",
    b"ban": "4b4acc0300",
    b"banana": "4b4acc034200",
    b"AAAAAAA": "73840000",
    bytes([0x2E, 0x20, 0x2E, 0x20, 0x2E, 0x20, 0x20]): "d35300410500",
}


@pytest.mark.parametrize("data", list(HAND), ids=[repr(k)[:20] for k in HAND])
def test_hand_derived(oc, data):
    st, got, _ = oc.deflate_compress(data)
    assert st == 0 and got.hex() == HAND[data] == statement(data).hex()
    assert zlib.decompress(got, -15) == data


def test_stored_block_of_high_bytes(oc):
    data = bytes(range(200, 256))
    st, got, _ = oc.deflate_compress(data)
    assert st == 0 and got == bytes([1, 56, 0, 0xC7, 0xFF]) + data


# DeflateCompressionTests.swift:29-85 compress these strings and round-trip them
REFERENCE_STRINGS = [b"ban", b"banana", b"abaaba", b"abracadabra", b"cabbage", b"baabaabac", b"AAAAAAA",
                     b"Ok, this is some plain text that should compress well enough", b"\x00" * 64]


@pytest.mark.parametrize("data", REFERENCE_STRINGS)
def test_reference_strings(oc, oracle, data):
    st, got, _ = oc.deflate_compress(data)
    assert st == 0 and got == statement(data)
    assert zlib.decompress(got, -15) == data
    ost, dec, _ = oracle.deflate_decompress(got)
    assert ost == 0 and dec == data


CASES = K.cases()


@pytest.mark.parametrize("name,data", CASES, ids=[c[0] for c in CASES])
def test_catalogue(oc, name, data):
    st, got, _ = oc.deflate_compress(data)
    assert st == 0 and got == statement(data), name
    assert zlib.decompress(got, -15) == data


def test_catalogue_edges_hold(oc):
    d = dict(CASES)
    assert oc.deflate_compress(d["tie_stored"])[1][0] == 1                  # a tie goes to stored
    assert oc.deflate_compress(d["tie_minus_one_static"])[1][0] & 7 == 3
    assert oc.deflate_compress(d["random_65530"])[1][0] == 1
    assert oc.deflate_compress(d["random_65531"])[1][0] & 7 == 3


@pytest.mark.parametrize("variant", ["lt_32768", "no_record_far", "record_inside", "strict_tie", "limit_n", "bucket"])
def test_near_misses_are_caught(variant):
    """each near miss of the statement gets at least one catalogue case wrong"""
    wrong = [name for name, data in CASES if statement(data, variant) != statement(data)]
    assert wrong, variant


def test_oracle_decoder_round_trip(oc, oracle):
    for name, data in CASES:
        st, got, _ = oc.deflate_compress(data)
        ost, dec, _ = oracle.deflate_decompress(got)
        assert ost == 0 and dec == data, name


def test_zlib_archive(oc):
    for data in [b"", b"banana", H.textlike(100000, 3)]:
        st, got, _ = oc.zlib_archive(data)
        assert st == 0 and got[:2] == b"\x78\xda" and got[-4:] == struct.pack(">I", zlib.adler32(data))
        assert got[2:-4] == oc.deflate_compress(data)[1] and zlib.decompress(got) == data


def gzip_header(comment, name, hcrc, text, os, mtime, extra):
    """the header GzipArchive.archive writes (GzipArchive.swift:126-226), from the Swift source"""
    flg = (16 if comment is not None else 0) | (8 if name is not None else 0) | (4 if extra else 0) | (2 if hcrc else 0) | int(text)
    h = bytes([0x1F, 0x8B, 8, flg]) + struct.pack("<I", 0 if mtime is None else mtime & 0xFFFFFFFF) + bytes([2, os])
    if extra:
        h += struct.pack("<H", sum(4 + len(e[2]) for e in extra))
        for si1, si2, b in extra:
            h += bytes([si1, si2]) + struct.pack("<H", len(b)) + b
    for t in (name, comment):
        if t is not None:
            h += t if t.endswith(b"\0") else t + b"\0"
    if hcrc:
        h += struct.pack("<H", zlib.crc32(h) & 0xFFFF)
    return h


GRID = [(c, nm, hc, tx, os, mt, ex)
        for c in (None, b"", b"comment \xe9")
        for nm in (None, b"file.txt", b"z\0")
        for hc in (False, True)
        for tx in (False, True)
        for os in (0, 3, 7, 11, 255)
        for mt in (None, 0, -1, -1700000000, 1700000000, 2**40 + 5)
        for ex in ([], [(65, 66, b"")], [(1, 2, b"xy"), (3, 4, bytes(300))])]


def test_gzip_header_grid(oc):
    data = H.textlike(5000, 9)
    body = oc.deflate_compress(data)[1]
    tail = struct.pack("<II", zlib.crc32(data), len(data))
    for c, nm, hc, tx, os, mt, ex in GRID[::7]:
        st, got, _ = oc.gzip_archive(data, comment=c, fileName=nm, writeHeaderCRC=hc, isTextFile=tx, osByte=os,
                                     modificationTime=mt, extraFields=ex)
        assert st == 0 and got == gzip_header(c, nm, hc, tx, os, mt, ex) + body + tail
        assert gzip.decompress(got) == data


def test_gzip_xlen_limit(oc):
    ok = [(1, 1, bytes(65531))]                       # XLEN 65 535
    st, got, _ = oc.gzip_archive(b"x", extraFields=ok)
    assert st == 0 and gzip.decompress(got) == b"x"
    st, _, _ = oc.gzip_archive(b"x", extraFields=[(1, 1, bytes(65532))])
    assert st == 607                                  # GzipError.cannotEncodeISOLatin1
    st, _, _ = oc.gzip_archive(b"x", extraFields=[(1, 1, bytes(30000)), (2, 2, bytes(35532))])
    assert st == 607
