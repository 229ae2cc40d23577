"""Multi-block .xz archives for the block-parallel XZ batch (swc_xz_block_unarchive_batch), and a Python restatement of the two
walks it relies on.

The batch finds every block from the streams' indexes, read backwards from the end of the unit (`back_walk`, the rule of
xz::back_stream in xz_framing.cuh), decodes the blocks side by side, and accepts a unit only when the reference's forward walk
agrees.  The cases here are the shapes multi-threaded `xz` writes (many independent blocks, size fields in the headers, every
check type, Delta chains, empty blocks and streams, stream padding) and the damaged ones where the two walks disagree:
swapped index records, a wrong record count, a look-alike index and footer inside a payload, a damaged header CRC, check or
block padding in block k.  `forward_blocks` restates where the forward walk finds the blocks, so the CPU test can show that
each disagreement case really gives block starts or sizes the forward walk does not.

Every case's status is the oracle's (tests/test_xz_block_cases_cpu.py pins that on the CPU)."""
import lzma
import struct

import helpers as H
import xz_cases as X
from test_framing_handmade import xz_block, xz_footer, xz_header, xz_index

OK, TRAP = 0, 2
XZ_MAGIC, XZ_FIELD, XZ_INFO_CRC, XZ_DATA_SIZE, XZ_CHECK, XZ_PADDING = 801, 802, 803, 806, 807, 808


def delta_encode(raw, dist):
    """the bytes DeltaFilter.swift:11-32 decodes to `raw`"""
    return bytes((raw[j] - (raw[j - dist] if j >= dist else 0)) & 0xFF for j in range(len(raw)))


def stream(blocks, check=X.CHECK_CRC32, sizes=None, edit=None, bad_check=None, bad_hdr_crc=None, bad_pad=None,
           filters=None):
    """one stream of blocks (payload, dictionary byte, decoded bytes).  sizes[k]: size fields in block k's header; edit(records)
    -> (records, count) rewrites the index; bad_check / bad_hdr_crc / bad_pad: the block whose check, header CRC or block
    padding is damaged; filters[k]: (filter list bytes, filter count) of block k"""
    body, records = b"", []
    for k, (payload, dict_byte, raw) in enumerate(blocks):
        filt, nf = filters[k] if filters and filters[k] else (b"\x21\x01" + bytes([dict_byte]), 1)
        ck = X.check_bytes(check, raw)
        if bad_check == k:
            ck = bytes([ck[0] ^ 0x40]) + ck[1:]
        with_sizes = sizes is not None and sizes[k]
        b, unpadded = xz_block(check, flags=nf - 1, comp=len(payload) if with_sizes else None,
                               uncomp=len(raw) if with_sizes else None, filt=filt, data=payload, check_bytes=ck,
                               bad_hdr_crc=bad_hdr_crc == k, block_pad_byte=7 if bad_pad == k else 0)
        body += b
        records.append((unpadded, len(raw)))
    count = None
    if edit is not None:
        records, count = edit(records)
    idx = xz_index(records, count)
    return xz_header(check) + body + idx + xz_footer(len(idx), check)


def own_blocks(m, size=3000, seed=120):
    """m distinct text blocks of about `size` bytes, each its own LZMA2 stream"""
    t = H.textlike(size * m + 7 * m, seed)
    out = []
    for k in range(m):
        raw = t[k * size:(k + 1) * size + k * 7 % 13]
        out.append((X.lzma2_raw(raw), 0x10, raw))
    return out


def lookalike(check=X.CHECK_CRC32):
    """-> (archive, cut): a one-block stream whose block is one uncompressed LZMA2 chunk carrying a look-alike index and footer
    that describe a stream from byte 0 to themselves.  The archive is valid; its first `cut` bytes end at the look-alike
    footer, where a backward walk finds a stream that covers the unit, while the forward walk runs into the chunk."""
    hdr_len = 12 + (1 + 1 + 3 + 4 + 3) // 4 * 4                  # stream header + block header (LZMA2 filter, no sizes)
    at = hdr_len + 3                                           # behind the uncompressed chunk's 3-byte header
    fill = (-at) % 4 + 8
    istart = at + fill
    fake_idx = xz_index([(istart - 12, 100)])
    fake = fake_idx + xz_footer(len(fake_idx), check)
    data = b"\x5A" * fill + fake + b"tail of the payload"
    payload = bytes([1]) + struct.pack(">H", len(data) - 1) + data + b"\x00"
    arc = stream([(payload, 0x10, data)], check)
    assert arc[istart:istart + len(fake)] == fake
    return arc, istart + len(fake)


_CASES = None


def cases():
    """-> [X.Arc] with expected statuses"""
    global _CASES
    if _CASES is not None:
        return _CASES
    out = []
    blocks = own_blocks(64)
    small = own_blocks(64, size=60, seed=121)
    for m in (1, 2, 3, 5, 8, 17, 33, 64):
        for sz in (False, True):
            out.append(X.Arc(f"{m} blocks, sizes {sz}", stream(blocks[:m], X.CHECK_CRC64, sizes=[sz] * m), OK))
    out.append(X.Arc("64 small blocks, alternating sizes", stream(small, X.CHECK_CRC32, sizes=[k % 2 == 0 for k in range(64)]), OK))
    for check in (X.CHECK_NONE, X.CHECK_CRC32, X.CHECK_CRC64, X.CHECK_SHA256):
        out.append(X.Arc(f"5 blocks, check {check}", stream(blocks[:5], check, sizes=[True, False] * 2 + [True]), OK))

    # Delta chains in front of LZMA2, one per block
    t = H.textlike(9000, 122)
    chains = [(1,), (4,), (256,), (2, 1), (32, 4, 1)]
    dblocks, dfilters = [], []
    for k, chain in enumerate(chains):
        raw = t[k * 1800:(k + 1) * 1800]
        enc = raw
        for d in chain:                                         # decode runs the listed Deltas last to first
            enc = delta_encode(enc, d)
        dblocks.append((X.lzma2_raw(enc), 0x10, raw))
        filt = b"".join(b"\x03\x01" + bytes([d - 1]) for d in chain) + b"\x21\x01\x10"
        dfilters.append((filt, len(chain) + 1))
    out.append(X.Arc("Delta chains, 5 blocks", stream(dblocks, X.CHECK_CRC64, filters=dfilters), OK))

    empty = (X.lzma2_raw(b""), 0x10, b"")
    out.append(X.Arc("0-byte blocks between others", stream([empty, blocks[0], empty, empty, blocks[1], empty]), OK))
    out.append(X.Arc("one 0-byte block", stream([empty], X.CHECK_SHA256), OK))
    zero = stream([], X.CHECK_CRC64)
    out.append(X.Arc("stream of zero blocks", zero, OK))
    s1, s2 = stream(blocks[:3], X.CHECK_CRC32, sizes=[True] * 3), stream(blocks[3:7], X.CHECK_SHA256)
    for pad in (0, 4, 8):
        p = bytes(pad)
        out.append(X.Arc(f"multi-stream, {pad} bytes of padding", s1 + p + zero + p + s2 + p + stream(blocks[7:9]) + p, OK))

    # the two walks disagree
    four = blocks[:1] + small[:1] + blocks[1:2] + small[1:2]
    swap = lambda i, j, f: lambda r: ([(r[j][0], r[i][1]) if k == i else (r[i][0], r[j][1]) if k == j else x
                                       for k, x in enumerate(r)] if f == 0 else
                                      [(r[i][0], r[j][1]) if k == i else (r[j][0], r[i][1]) if k == j else x
                                       for k, x in enumerate(r)], None)
    out.append(X.Arc("unpadded sizes of blocks 0 and 1 swapped", stream(four, edit=swap(0, 1, 0)), XZ_FIELD))
    out.append(X.Arc("unpadded sizes of blocks 1 and 3 swapped", stream(four, edit=swap(1, 3, 0)), XZ_FIELD))
    out.append(X.Arc("decoded sizes of blocks 0 and 1 swapped", stream(four, edit=swap(0, 1, 1)), XZ_DATA_SIZE))
    out.append(X.Arc("decoded sizes of blocks 2 and 3 swapped", stream(four, edit=swap(2, 3, 1)), XZ_DATA_SIZE))
    out.append(X.Arc("record count one high", stream(four, edit=lambda r: (r, len(r) + 1)), XZ_FIELD))
    out.append(X.Arc("record count one low", stream(four, edit=lambda r: (r, len(r) - 1)), XZ_FIELD))
    out.append(X.Arc("one record too few", stream(four, edit=lambda r: (r[:-1], None)), XZ_FIELD))
    arc, cut = lookalike()
    out.append(X.Arc("look-alike index and footer inside a payload", arc, OK))
    out.append(X.Arc("cut at the look-alike footer", arc[:cut], TRAP))
    out.append(X.Arc("look-alike stream behind a real one, cut at its footer", s1 + arc[:cut], TRAP))
    for k in (0, 2, 3):
        out.append(X.Arc(f"header CRC of block {k} of 4", stream(four, bad_hdr_crc=k), XZ_INFO_CRC))
        out.append(X.Arc(f"check of block {k} of 4", stream(four, X.CHECK_CRC64, bad_check=k), XZ_CHECK))
    pad_k = [k for k, b in enumerate(four) if (len(b[0]) + 12) % 4][0]
    out.append(X.Arc(f"non-zero block padding in block {pad_k}", stream(four, bad_pad=pad_k), XZ_PADDING))
    names = [a.name for a in out]
    assert len(set(names)) == len(names)
    _CASES = out
    return out


# ---- the two walks, restated ---------------------------------------------------------------------------------------------
def _vli(b, o, end):
    v, i = 0, 0
    while True:
        if o >= end or i >= 9:
            return None, o
        c = b[o]
        o += 1
        v |= (c & 0x7F) << (7 * i)
        i += 1
        if c < 0x80:
            return (v, o) if i == 1 or c else (None, o)


def back_walk(b):
    """-> [(start, decoded size, output offset)] of every block, in order, as the backward walk from the end finds them, or
    None when it does not reach byte 0 (xz::back_stream / xz::declared_size)"""
    pos, streams = len(b), []
    while pos > 0:
        while pos >= 4 and b[pos - 4:pos] == bytes(4):
            pos -= 4
        if pos < 32 or b[pos - 2:pos] != b"YZ":
            return None
        foot = pos - 12
        isize = (struct.unpack("<I", b[foot + 4:foot + 8])[0] + 1) * 4
        if isize + 12 > foot:
            return None
        istart = foot - isize
        if b[istart] != 0:
            return None
        count, o = _vli(b, istart + 1, foot)
        if count is None or count > 1000000:
            return None
        recs, total = [], 0
        for _ in range(count):
            unp, o = _vli(b, o, foot)
            unc, o = _vli(b, o, foot) if unp is not None else (None, o)
            if unp is None or unc is None or unp <= 0 or unp > istart:
                return None
            padded = (unp + 3) & ~3
            if padded > istart - total:
                return None
            total += padded
            recs.append((padded, unc))
        if total + 12 > istart:
            return None
        start = istart - total - 12
        if b[start:start + 6] != b"\xFD7zXZ\x00":
            return None
        streams.append((start, recs))
        pos = start
    out, at = [], 0
    for start, recs in reversed(streams):
        o = start + 12
        for padded, unc in recs:
            out.append((o, unc, at))
            o += padded
            at += unc
    return out


def _skim(b, o):
    """-> (end, decoded size) of the LZMA2 stream at o, by its chunk headers, or None when it runs off the data"""
    n = 0
    while o < len(b):
        c = b[o]
        if c == 0:
            return o + 1, n
        if c in (1, 2):
            if o + 3 > len(b):
                return None
            size = (b[o + 1] << 8 | b[o + 2]) + 1
            o, n = o + 3 + size, n + size
            continue
        if o + 5 > len(b):
            return None
        n += ((c & 0x1F) << 16 | b[o + 1] << 8 | b[o + 2]) + 1
        o += 5 + ((c & 0x60) >> 5 >= 2) + (b[o + 3] << 8 | b[o + 4]) + 1
    return None


def forward_blocks(b):
    """-> [(start, decoded size)] of the blocks the forward walk reaches, in order, up to the first block or stream it cannot
    parse (block headers, LZMA2 chunk headers and padding only: no CRC is checked)"""
    out, o = [], 0
    while o + 12 <= len(b) and b[o:o + 6] == b"\xFD7zXZ\x00":
        csize = {0: 0, 1: 4, 4: 8, 10: 32}.get(b[o + 7] & 0xF, 0)
        o += 12
        while o < len(b) and b[o] != 0:
            start, hsize = o, (b[o] + 1) * 4
            if start + hsize > len(b):
                return out
            s = _skim(b, start + hsize)
            if s is None:
                return out
            end, n = s
            out.append((start, n))
            o = end + (-(end - start) % 4) + csize
        if o >= len(b):
            return out
        count, p = _vli(b, o + 1, len(b))
        if count is None:
            return out
        for _ in range(2 * count):
            _, p = _vli(b, p, len(b))
            if _ is None:
                return out
        p += (-(p - o) % 4) + 4 + 12                          # index padding and CRC, footer
        while p + 4 <= len(b) and b[p:p + 4] == bytes(4):
            p += 4
        o = p
    return out


def liblzma(data):
    """the file decoded by liblzma, stream by stream, skipping stream padding (Python's lzma.decompress stops at padding)"""
    out = b""
    while data:
        d = lzma.LZMADecompressor(format=lzma.FORMAT_XZ)
        out += d.decompress(data)
        assert d.eof
        data = d.unused_data
        while data[:4] == bytes(4):
            data = data[4:]
    return out
