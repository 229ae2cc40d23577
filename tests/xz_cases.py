"""A named catalogue of .xz archives for the batched XZ decoder (swc_xz_unarchive_batch): the golden fixtures, the hand-derived
framing cases of test_framing_handmade, Python's lzma at every check type, preset and Delta chain, check fields around the
SHA-256 padding edges and the warp CRC's lane segments, hand-framed multi-block and multi-stream archives built from the raw
LZMA2 streams of lzma_cases, stream padding, wrong checks, short units and the filter chains the batch does not run.

Every archive's expected status and output are the oracle's (tests/test_xz_cases_cpu.py pins that on the CPU).  The one
exception is `unsupported`: the archives whose first failing point is a filter chain or an LZMA chunk the batch does not run
(DESIGN §6), for which the batch answers SWC_ERR_UNSUPPORTED while the oracle and swc_xz_unarchive decode on."""
import hashlib
import lzma
import random
import struct
import zlib

import helpers as H
import lzma_cases as LC
import lzma_writer as W
from test_framing_handmade import GOOD, xz_block, xz_cases, xz_footer, xz_header, xz_index

OK, OVERFLOW, TRAP, UNSUPPORTED = 0, 1, 2, 6
XZ_MAGIC, XZ_FIELD, XZ_CHECK, XZ_PADDING = 801, 802, 807, 808
PAYLOAD_CARRYING = (XZ_CHECK,)
CHECK_NONE, CHECK_CRC32, CHECK_CRC64, CHECK_SHA256 = 0, 1, 4, 10
CHECK_IDS = {CHECK_NONE: lzma.CHECK_NONE, CHECK_CRC32: lzma.CHECK_CRC32, CHECK_CRC64: lzma.CHECK_CRC64,
             CHECK_SHA256: lzma.CHECK_SHA256}


class Arc:
    """`unsupported_at`: for an archive the batch refuses, the length from which a cut of it reaches the refused point (the
    block's first data byte for a filter chain, the fifth range-coder byte of the chunk for lc + lp > 4): shorter cuts fail
    earlier, exactly as in the reference"""
    __slots__ = ("name", "data", "status", "unsupported_at")

    def __init__(self, name, data, status=None, unsupported_at=None):
        self.name, self.data, self.status, self.unsupported_at = name, bytes(data), status, unsupported_at

    @property
    def unsupported(self):
        return self.unsupported_at is not None


def crc64(data):
    """CRC-64/XZ, bitwise (ECMA-182 reflected)"""
    c = 0xFFFFFFFFFFFFFFFF
    for b in data:
        c ^= b
        for _ in range(8):
            c = (c >> 1) ^ 0xC96C5795D7870F42 if c & 1 else c >> 1
    return c ^ 0xFFFFFFFFFFFFFFFF


def check_bytes(check, raw):
    if check == CHECK_NONE:
        return b""
    if check == CHECK_CRC32:
        return struct.pack("<I", zlib.crc32(raw))
    if check == CHECK_CRC64:
        return struct.pack("<Q", crc64(raw))
    return hashlib.sha256(raw).digest()


def lzma2_raw(raw, preset=1, dict_size=1 << 16):
    return lzma.compress(raw, format=lzma.FORMAT_RAW, filters=[{"id": lzma.FILTER_LZMA2, "preset": preset, "dict_size": dict_size}])


def framed(blocks, check=CHECK_CRC32, sizes=None, bad_check=None):
    """one hand-framed stream of blocks (payload, dictionary byte, decoded bytes[, filter list bytes, filter count]);
    sizes[k]: write the size fields in block k's header; bad_check: the index of a block whose check field is damaged"""
    body, records = b"", []
    for k, blk in enumerate(blocks):
        payload, dict_byte, raw = blk[:3]
        filt, nfilters = blk[3:] if len(blk) > 3 else (b"\x21\x01" + bytes([dict_byte]), 1)
        flags = nfilters - 1
        ck = check_bytes(check, raw)
        if bad_check == k:
            ck = bytes([ck[0] ^ 0x40]) + ck[1:]
        with_sizes = sizes is not None and sizes[k]
        b, unpadded = xz_block(check, flags=flags, comp=len(payload) if with_sizes else None,
                               uncomp=len(raw) if with_sizes else None, filt=filt, data=payload, check_bytes=ck)
        body += b
        records.append((unpadded, len(raw)))
    idx = xz_index(records)
    return xz_header(check) + body + idx + xz_footer(len(idx), check)


def python_lzma(raw, check, preset=1, deltas=()):
    filters = [{"id": lzma.FILTER_DELTA, "dist": d} for d in deltas] + [{"id": lzma.FILTER_LZMA2, "preset": preset}]
    return lzma.compress(raw, format=lzma.FORMAT_XZ, check=CHECK_IDS[check], filters=filters)


def lzma2_blocks():
    """(payload, dictionary byte, decoded bytes) of every lzma_cases LZMA2 stream the batch decodes (batch status 0)"""
    return [(c.data, c.dict_byte, c.model.out) for c in LC.catalogue() if c.form == "lzma2" and c.batch == W.OK]


def wide_chunk(stream):
    """offset of the first LZMA chunk with lc + lp > 4 in an LZMA2 stream"""
    o = 0
    while stream[o] != 0:
        c = stream[o]
        if c in (1, 2):
            o += 3 + (stream[o + 1] << 8 | stream[o + 2]) + 1
            continue
        if (c & 0x60) >> 5 >= 2:
            b = stream[o + 5]
            if b % 9 + (b // 9) % 5 > 4:
                return o
        o += 5 + ((c & 0x60) >> 5 >= 2) + (stream[o + 3] << 8 | stream[o + 4]) + 1
    raise ValueError("no chunk with lc + lp > 4")


_CASES = None


def cases():
    global _CASES
    if _CASES is not None:
        return _CASES
    out = []
    for rel, _ in H.fixtures("XZ/"):
        out.append(Arc(f"fixture {rel}", H.fixture(rel), OK))
    for name, blob, st in xz_cases():
        out.append(Arc(f"framing {name}", blob, st))

    text = H.textlike(20000, 90)
    for check in CHECK_IDS:
        for preset in (0, 6, 9 | lzma.PRESET_EXTREME):
            out.append(Arc(f"python check {check} preset {preset}", python_lzma(text, check, preset), OK))
        for deltas in ((1,), (2,), (4,), (32,), (256,), (1, 2), (4, 256), (32, 2, 1)):
            out.append(Arc(f"python check {check} delta {deltas}", python_lzma(text[:7000], check, 1, deltas), OK))
    rng_raw = H.random_bytes(random.Random(91), 3000)
    for check in (CHECK_CRC32, CHECK_CRC64, CHECK_SHA256):
        for n in (0, 1, 15, 16, 17, 54, 55, 56, 57, 63, 64, 65, 119, 120, 121, 127, 128, 129, 511, 512, 513, 1023, 1024, 1025,
                  32 * 16 * 3 - 1, 32 * 16 * 3, 32 * 16 * 3 + 1, 2047, 2048, 2049, 2999):
            out.append(Arc(f"check {check} size {n}", python_lzma(rng_raw[:n], check), OK))

    # hand-framed multi-block streams of the lzma_cases streams, with and without size fields
    blocks = lzma2_blocks()
    t = H.textlike(60000, 92)
    own = [(lzma2_raw(t[k * 3000:(k + 1) * 3000 + k * 7]), 0x10, t[k * 3000:(k + 1) * 3000 + k * 7]) for k in range(20)]
    for m in (1, 2, 3, 7, 20):
        for check in (CHECK_CRC32, CHECK_CRC64):
            out.append(Arc(f"framed {m} blocks check {check}", framed(own[:m], check, sizes=[k % 2 == 0 for k in range(m)]), OK))
    for j in range(0, len(blocks), 12):
        group = blocks[j:j + 12]
        out.append(Arc(f"framed lzma_cases {j}..{j + len(group) - 1}", framed(group, CHECK_CRC64 if j % 24 else CHECK_CRC32,
                                                                             sizes=[k % 3 == 1 for k in range(len(group))]), OK))

    # multi-stream files and stream padding
    s1, s2, s3 = framed(own[:2]), python_lzma(t[:5000], CHECK_CRC64), python_lzma(t[5000:9000], CHECK_SHA256)
    for pad in (0, 4, 8):
        out.append(Arc(f"three streams, {pad} bytes of padding", s1 + bytes(pad) + s2 + bytes(pad) + s3, OK))
    for pad in (1, 2, 3):
        out.append(Arc(f"two streams, bad padding of {pad}", s1 + bytes(pad) + s2, XZ_PADDING))
    out.append(Arc("two streams, non-zero byte inside the padding", s1 + b"\0\0\x01\0" + s2, XZ_PADDING))
    out.append(Arc("stream, 8 trailing zero bytes", s2 + bytes(8), OK))

    # a wrong check in block k of m
    for check in (CHECK_CRC32, CHECK_CRC64, CHECK_SHA256):
        for k in (0, 2, 4):
            out.append(Arc(f"wrong check {check} in block {k} of 5", framed(own[:5], check, bad_check=k), XZ_CHECK))
    out.append(Arc("wrong check in the second stream", s1 + framed(own[2:4], CHECK_CRC64, bad_check=1), XZ_CHECK))

    # short units and short tails
    out.append(Arc("empty unit", b"", OK))
    for n in range(1, 32):
        out.append(Arc(f"{n}-byte unit", GOOD[:n], XZ_MAGIC))
    for n in (1, 5, 31):
        out.append(Arc(f"stream and {n} non-zero bytes", GOOD + b"\x07" * n, XZ_MAGIC))

    # a block never sees earlier blocks' bytes (a new LZMA2Decoder per block): a block whose first chunk resets the state but
    # not the dictionary, then reaches back, fails even though the blocks before it decoded
    for name, ops in (("a rep", [W.rep(0, 2)]), ("a match behind its start", LC.lits(b"ab") + [W.match(8, 150)]),
                      ("a short rep", [W.SHORT])):
        c = LC.lzma2(name, 0, [W.Chunk(ops, reset=2, props=(3, 0, 2))], dict_byte=0x10)
        out.append(Arc(f"block 3 of 3 opens with {name} and no dictionary reset",
                       framed(own[:2] + [(c.data, 0x10, c.model.out)]), c.model.status))

    # filter chains and LZMA chunks the batch does not run, each after valid blocks; and the same archives failing earlier
    pl = lzma2_raw(t[:4000])
    two = own[:1] + [(pl, 0x10, t[:4000], b"\x21\x01\x10\x21\x01\x10", 2)]
    last = own[:2] + [(pl, 0x10, t[:4000], b"\x21\x01\x10\x03\x01\x00", 2)]
    for name, blocks in (("two LZMA2 filters", two), ("Delta filter last", last)):
        data = framed(blocks)
        out.append(Arc(name, data, unsupported_at=data.index(pl)))
        out.append(Arc(f"{name}, wrong check in the block before", framed(blocks, bad_check=len(blocks) - 2), XZ_CHECK))
    wide = [c for c in LC.catalogue() if c.name == "l2_props_lc4_lp1_after_small"][0]
    blocks = own[:1] + [(wide.data, wide.dict_byte, wide.model.out)] + own[1:2]
    data = framed(blocks)
    out.append(Arc("lc + lp > 4 chunk in block 2 of 3", data, unsupported_at=data.index(wide.data) + wide_chunk(wide.data) + 6 + 5))
    out.append(Arc("lc + lp > 4 chunk in block 2 of 3, wrong check in block 1", framed(blocks, bad_check=0), XZ_CHECK))
    names = [a.name for a in out]
    assert len(set(names)) == len(names)
    _CASES = out
    return out


def expected(oracle, arc, cut=None):
    """-> (status, output) the batch must give for the archive, or for its first `cut` bytes: the oracle's, or
    SWC_ERR_UNSUPPORTED with no output once the refused point is reached"""
    data = arc.data if cut is None else arc.data[:cut]
    if arc.unsupported and len(data) >= arc.unsupported_at:
        return UNSUPPORTED, b""
    st, out, _ = oracle.xz_unarchive(data)
    return st, out if st in (OK,) + PAYLOAD_CARRYING else b""
