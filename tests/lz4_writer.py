"""Test-only LZ4 block and frame writer, and a model of the reference's decoder.

The writer lays a block out from explicit sequences and lets every field be what no encoder writes: the token's two
nibbles, the length-extension bytes (a run that ends in 255, or runs off the block), the raw offset bytes, the final
literal run or none at all.  The frame builders write independent, dependent and legacy frames whose blocks may be stored,
empty, carry a (possibly wrong) block checksum, and whose descriptor may hold a content size, a content checksum and a
dictionary ID.

The expected answer is not taken from the oracle: `decode_block` restates process(block:_:) of Sources/LZ4/LZ4.swift
(:332-413) and `decode` / `multi_decode` restate decompress / multiDecompress and the frame walks (:73-330), including
the `out.isEmpty` rule that gives a dependent frame's first block the dictionary and every later one the last 64 KiB of
the frame's output.  Each decoded sequence is recorded in a trace for the coverage assertions."""
import struct

import oracle_xxh

OK, OVERFLOW = 0, 1
TRUNCATED, CORRUPTED, CHECKSUM, UNSUPPORTED = 501, 502, 503, 504

FRAME_MAGIC, LEGACY_MAGIC = 0x184D2204, 0x184C2102
WINDOW = 64 * 1024
BLOCK_SIZES = {0x40: 64 << 10, 0x50: 256 << 10, 0x60: 1 << 20, 0x70: 4 << 20}


def ext(v):
    """the canonical extension bytes of a length field value `v` >= 0 (the part past the nibble's 15)"""
    return b"\xFF" * (v // 255) + bytes([v % 255])


class Seq:
    """One sequence.  `mlen` None: the final, literal-only sequence.  Overrides are written verbatim: `lit_nib` / `ml_nib`
    the token's nibbles, `lit_ext` / `ml_ext` the extension bytes, `off_raw` the offset field (any number of bytes)."""
    __slots__ = ("lit", "mlen", "offset", "lit_nib", "lit_ext", "off_raw", "ml_nib", "ml_ext")

    def __init__(self, lit=b"", mlen=None, offset=None, lit_nib=None, lit_ext=None, off_raw=None, ml_nib=None, ml_ext=None):
        self.lit, self.mlen, self.offset = bytes(lit), mlen, offset
        self.lit_nib, self.lit_ext, self.off_raw, self.ml_nib, self.ml_ext = lit_nib, lit_ext, off_raw, ml_nib, ml_ext

    def encode(self):
        n = len(self.lit)
        lnib = min(n, 15) if self.lit_nib is None else self.lit_nib
        lext = self.lit_ext if self.lit_ext is not None else (ext(n - 15) if lnib == 15 else b"")
        if self.mlen is None:
            return bytes([lnib << 4]) + lext + self.lit
        m = self.mlen - 4
        mnib = min(m, 15) if self.ml_nib is None else self.ml_nib
        mext = self.ml_ext if self.ml_ext is not None else (ext(m - 15) if mnib == 15 else b"")
        off = self.off_raw if self.off_raw is not None else struct.pack("<H", self.offset)
        return bytes([lnib << 4 | mnib]) + lext + self.lit + off + mext


def write_block(seqs):
    return b"".join(s.encode() for s in seqs)


def block(seqs, last=b""):
    """a canonical block: (literals, match length, offset) sequences, then the final literal run (None: no final sequence)"""
    out = [Seq(l, m, o) for l, m, o in seqs]
    if last is not None:
        out.append(Seq(last))
    return write_block(out)


class Result:
    __slots__ = ("status", "out", "trace", "nseq", "max_lit", "max_mlen")

    def __init__(self):
        self.status, self.out, self.trace, self.nseq, self.max_lit, self.max_mlen = OK, b"", [], 0, 0, 0

    def __repr__(self):
        return f"Result(status={self.status}, out={len(self.out)} bytes, nseq={self.nseq})"


class _Fail(Exception):
    def __init__(self, code):
        super().__init__(code)
        self.code = code


def decode_block(data, dictionary=None):
    """process(block: data, dictionary) of LZ4.swift:332-413 -> Result.  The output is what the reference returns: the
    block's bytes without the dictionary, nothing when it throws.  Trace entries:
      ("ext", field, start position mod 32, bytes in the run, whether the run ended inside the block)
      ("lit", sequence index, literal count)
      ("match", sequence index, block output position, offset, match length, offset - out.endIndex, source kind,
       offset < match length, whether the source reads the previous match's output)   source kind: "out", "dict",
       "straddle" (starts in the dictionary, ends in the block's output)
      ("offset", offset - out.endIndex) for a rejected offset, ("trunc", field) for a block that ends inside `field`,
      ("end", rule, final literal count, out.endIndex - lastMatchStartIndex or None)"""
    r = Result()
    d = bytes(dictionary or b"")
    out = bytearray(d)                                              # :334
    out_start = len(out)                                            # :335
    n = len(data)
    ip = 0
    seq_count = 0                                                   # :338
    last_match_start = -1                                           # :339
    prev_match = None                                               # (start, end) of the previous match's output

    def extension(field, value):
        nonlocal ip
        start, count = ip, 0
        while True:                                                 # :349-362 / :387-400
            if n - ip < 1:
                r.trace.append(("ext", field, start % 32, count, False))
                r.trace.append(("trunc", field + "_ext"))
                raise _Fail(TRUNCATED)
            b = data[ip]
            ip += 1
            count += 1
            value += b                                              # Int overflow needs > 2^55 input bytes
            if b != 255:
                r.trace.append(("ext", field, start % 32, count, True))
                return value

    try:
        while True:
            seq_count += 1                                          # :342
            if n - ip < 1:                                          # :343
                r.trace.append(("trunc", "token"))
                raise _Fail(TRUNCATED)
            token = data[ip]
            ip += 1
            lit = token >> 4                                        # :347
            if lit == 15:
                lit = extension("lit", lit)
            if n - ip < lit:                                        # :364
                r.trace.append(("trunc", "lits"))
                raise _Fail(TRUNCATED)
            out += data[ip:ip + lit]                                # :366
            ip += lit
            r.nseq = seq_count
            r.max_lit = max(r.max_lit, lit)
            r.trace.append(("lit", seq_count - 1, lit))
            if ip == n:                                             # :369 reader.isFinished
                dist = None if last_match_start == -1 else len(out) - last_match_start
                if not (lit >= 5 or seq_count == 1):                # :371
                    r.trace.append(("end", "short_literals", lit, dist))
                    raise _Fail(CORRUPTED)
                if not (last_match_start == -1 or dist >= 12):      # :373
                    r.trace.append(("end", "match_near_end", lit, dist))
                    raise _Fail(CORRUPTED)
                r.trace.append(("end", "single" if seq_count == 1 else "ok", lit, dist))
                break
            if n - ip < 2:                                          # :378
                r.trace.append(("trunc", "offset"))
                raise _Fail(TRUNCATED)
            offset = data[ip] | data[ip + 1] << 8                   # :380
            ip += 2
            if not (offset > 0 and offset <= len(out)):             # :382
                r.trace.append(("offset", offset - len(out)))
                raise _Fail(CORRUPTED)
            mlen = 4 + (token & 15)                                 # :385
            if mlen == 19:
                mlen = extension("mlen", mlen)
            last_match_start = len(out)                             # :405
            src = len(out) - offset                                 # :406
            kind = "out" if src >= out_start else ("dict" if src + min(mlen, offset) <= out_start else "straddle")
            dep = prev_match is not None and src < prev_match[1] and src + min(mlen, offset) > prev_match[0]
            r.trace.append(("match", seq_count - 1, len(out) - out_start, offset, mlen, offset - len(out), kind,
                            offset < mlen, dep))
            if offset >= mlen:                                      # :407-409, a byte at a time in the reference
                out += out[src:src + mlen]
            else:
                period = out[src:]
                out += (period * (mlen // offset + 1))[:mlen]
            prev_match = (last_match_start, len(out))
            r.max_mlen = max(r.max_mlen, mlen)
    except _Fail as e:
        r.status = e.code
        return r
    r.out = bytes(out[out_start:])                                  # :412
    return r


# ------------------------------------------------------------------------------------------------------- kernel window
def kernel_window_runs(data, dict_len=0):
    """Where the one-kernel decoder (lz4_block_body in swcompression_b200/csrc/lz4.cu) sees each length-extension run of a
    block that starts a unit, as a restatement of its Window: a 32-byte window of the block that `ensure(at, need)`
    re-bases at `at` whenever [at, at + need) leaves it -- for the token (need 1), the offset (need 2) and each pass of
    read_extension (need 1).  This describes the kernel, not the reference, and is kept apart from decode_block; it
    stops where the kernel's walk stops (a cut, or an offset past the dictionary and the output so far).
    -> [(field, window lane of the run's first byte, bytes in the run, whether the run ends past that window)]"""
    n, base, ip, op, runs = len(data), 0, 0, 0, []

    def ensure(at, need):
        nonlocal base
        if at < base or at + need > base + 32:
            base = at

    def extension(field):
        nonlocal ip
        start, lane = ip, None
        while True:
            if ip >= n:
                return None
            ensure(ip, 1)
            pos = ip - base
            lane = pos if lane is None else lane
            end = next((j for j in range(pos, 32) if base + j >= n or data[base + j] != 255), None)
            if end is None:                                     # every lane from pos on holds 255: the next window
                ip = base + 32
                continue
            if base + end >= n:
                return None
            ip = base + end + 1
            runs.append((field, lane, ip - start, lane + ip - start > 32))
            return sum(data[start:ip])

    while ip < n:
        ensure(ip, 1)
        token = data[ip]
        ip += 1
        lit = token >> 4
        if lit == 15:
            lit = extension("lit")
            if lit is None:
                break
            lit += 15
        if n - ip < lit:
            break
        op += lit
        ip += lit
        if ip == n or n - ip < 2:
            break
        ensure(ip, 2)
        offset = data[ip] | data[ip + 1] << 8
        ip += 2
        if offset == 0 or offset > op + dict_len:
            break
        mlen = 4 + (token & 15)
        if mlen == 19:
            mlen = extension("mlen")
            if mlen is None:
                break
            mlen += 19
        op += mlen
    return runs


# --------------------------------------------------------------------------------------------------------------- frames
class FBlock:
    """One frame block: `data` the payload, `stored` the mark's high bit, `ck` the block checksum to write (None: the true
    one), `size` the mark's size field (None: len(data))."""
    __slots__ = ("data", "stored", "ck", "size")

    def __init__(self, data, stored=False, ck=None, size=None):
        self.data, self.stored, self.ck, self.size = bytes(data), stored, ck, size


def frame(blocks, independent=False, block_checksums=False, content_size=None, content_checksum=None, dict_id=None,
          bd=0x70, end=True):
    """An LZ4 frame.  `content_size` / `dict_id`: the descriptor fields (None: absent); `content_checksum`: the checksum
    word after the EndMark (None: absent; a bytes object: the checksum of those bytes; an int: that word)."""
    flg = 0x40 | (0x20 if independent else 0) | (0x10 if block_checksums else 0) | (0x08 if content_size is not None else 0)
    flg |= (0x04 if content_checksum is not None else 0) | (0x01 if dict_id is not None else 0)
    desc = bytes([flg, bd])
    if content_size is not None:
        desc += struct.pack("<Q", content_size)
    if dict_id is not None:
        desc += struct.pack("<I", dict_id)
    out = bytearray(struct.pack("<I", FRAME_MAGIC) + desc + bytes([(oracle_xxh.xxh32(desc) >> 8) & 0xFF]))
    for b in blocks:
        size = len(b.data) if b.size is None else b.size
        out += struct.pack("<I", size | (0x80000000 if b.stored else 0)) + b.data
        if block_checksums:
            out += struct.pack("<I", oracle_xxh.xxh32(b.data) if b.ck is None else b.ck)
    if end:
        out += struct.pack("<I", 0)
        if isinstance(content_checksum, (bytes, bytearray)):
            out += struct.pack("<I", oracle_xxh.xxh32(content_checksum))
        elif content_checksum is not None:
            out += struct.pack("<I", content_checksum)
    return bytes(out)


def legacy_frame(blocks):
    out = bytearray(struct.pack("<I", LEGACY_MAGIC))
    for b in blocks:
        out += struct.pack("<I", len(b)) + b
    return bytes(out)


def _u32(data, at):
    return struct.unpack_from("<I", data, at)[0]


def _is_magic(v):
    return v in (FRAME_MAGIC, LEGACY_MAGIC) or 0x184D2A50 <= v <= 0x184D2A5F


class FrameResult:
    """`status`, `out` (the frame's bytes; with CHECKSUM the bytes the error carries), `next` the offset after the frame,
    `blocks` the Result of every decoded block in order"""
    __slots__ = ("status", "out", "next", "blocks")

    def __init__(self, status, out, nxt, blocks):
        self.status, self.out, self.next, self.blocks = status, out, nxt, blocks


def _legacy(data, pos):
    """process(legacyFrame:) :160-186; `pos` is right after the magic"""
    out, blocks = bytearray(), []
    while pos < len(data):                                          # :164 !reader.isFinished
        if len(data) - pos < 4:
            return FrameResult(TRUNCATED, b"", pos, blocks)
        raw = _u32(data, pos)
        pos += 4
        if _is_magic(raw):                                          # :168-171
            pos -= 4
            break
        if len(data) - pos < raw:                                   # :177
            return FrameResult(TRUNCATED, b"", pos, blocks)
        r = decode_block(data[pos:pos + raw])                       # :183, no dictionary
        pos += raw
        blocks.append(r)
        if r.status:
            return FrameResult(r.status, b"", pos, blocks)
        out += r.out
    return FrameResult(OK, bytes(out), pos, blocks)


def _frame(data, pos, dictionary, ext_id):
    """process(frame:_:_:) :188-330; `pos` is right after the magic"""
    blocks = []

    def fail(code):
        return FrameResult(code, b"", pos, blocks)

    if len(data) - pos < 7:                                         # :191
        return fail(TRUNCATED)
    start = pos
    flg = data[pos]
    pos += 1
    if not ((flg & 0xC0) >> 6 == 1 and flg & 0x2 == 0):             # :198
        return fail(CORRUPTED)
    independent, block_ck, csize_p, cck, dictid_p = flg & 0x20, flg & 0x10, flg & 0x08, flg & 0x04, flg & 0x01
    bd = data[pos]
    pos += 1
    if bd not in BLOCK_SIZES:                                       # :216-228
        return fail(CORRUPTED)
    max_block = BLOCK_SIZES[bd]
    content_size = None
    if csize_p:
        if len(data) - pos < 13:                                    # :234
            return fail(TRUNCATED)
        content_size = struct.unpack_from("<Q", data, pos)[0]
        pos += 8
        if content_size >= 1 << 63:                                 # :240
            return fail(UNSUPPORTED)
    did = None
    if dictid_p:
        if dictionary is None:                                      # :250
            return fail(CORRUPTED)
        if len(data) - pos < 9:                                     # :254
            return fail(TRUNCATED)
        did = _u32(data, pos)
        pos += 4
    if ext_id is not None and did is not None and ext_id != did:    # :266-270
        return fail(CORRUPTED)
    hc = oracle_xxh.xxh32(data[start:pos])                          # :272-275
    if (hc >> 8) & 0xFF != data[pos]:
        return fail(CORRUPTED)
    pos += 1
    out = bytearray()
    while True:                                                     # :278
        if len(data) - pos < 4:
            return fail(TRUNCATED)
        mark = _u32(data, pos)
        pos += 4
        if mark == 0:                                               # :284
            break
        compressed = mark & 0x80000000 == 0
        size = mark & 0x7FFFFFFF
        if size > max_block:                                        # :292
            return fail(CORRUPTED)
        if len(data) - pos < size + (4 if block_ck else 0) + 4:     # :295
            return fail(TRUNCATED)
        bdata = data[pos:pos + size]
        pos += size
        if block_ck:                                                # :300
            ck = _u32(data, pos)
            pos += 4
            if oracle_xxh.xxh32(bdata) != ck:
                return fail(CORRUPTED)
        if compressed:
            if independent:                                         # :304-305
                r = decode_block(bdata, dictionary)
            elif not out and dictionary is not None:                # :307-309
                r = decode_block(bdata, bytes(dictionary)[-WINDOW:])
            else:                                                   # :311-312
                r = decode_block(bdata, bytes(out[-WINDOW:]))
            blocks.append(r)
            if r.status:
                return fail(r.status)
            out += r.out
        else:
            out += bdata                                            # :316
    if csize_p and len(out) != content_size:                        # :319-321
        return fail(CORRUPTED)
    if cck:
        if len(data) - pos < 4:                                     # :324
            return fail(TRUNCATED)
        ck = _u32(data, pos)
        pos += 4
        if oracle_xxh.xxh32(bytes(out)) != ck:                      # :326
            return FrameResult(CHECKSUM, bytes(out), pos, blocks)
    return FrameResult(OK, bytes(out), pos, blocks)


def _skippable(data, pos):
    """process(skippableFrame:) :148-155 -> (status, frame size after the magic)"""
    if len(data) - pos < 4:
        return TRUNCATED, 0
    size = _u32(data, pos)
    if len(data) - pos < size + 4:
        return TRUNCATED, 0
    return OK, size + 4


def decode(data, dictionary=None, dict_id=None):
    """LZ4.decompress(data:dictionary:dictionaryID:) :73-91 -> FrameResult"""
    data = bytes(data)
    pos = 0
    while True:
        if len(data) - pos < 4:                                     # :75
            return FrameResult(TRUNCATED, b"", pos, [])
        magic = _u32(data, pos)
        if magic == FRAME_MAGIC:
            return _frame(data, pos + 4, dictionary, dict_id)
        if 0x184D2A50 <= magic <= 0x184D2A5F:                       # :83-85: the rest, without the dictionary
            st, size = _skippable(data, pos + 4)
            if st:
                return FrameResult(st, b"", pos, [])
            pos += 4 + size
            dictionary, dict_id = None, None
            continue
        if magic == LEGACY_MAGIC:
            return _legacy(data, pos + 4)
        return FrameResult(CORRUPTED, b"", pos, [])


def multi_decode(data, dictionary=None, dict_id=None):
    """LZ4.multiDecompress :116-146 -> (status, list of the frames' outputs; with CHECKSUM the failing frame's last)"""
    data = bytes(data)
    result, pos = [], 0
    while True:
        if pos + 4 > len(data):                                     # :123
            return TRUNCATED, result
        magic = _u32(data, pos)
        pos += 4
        if magic == FRAME_MAGIC:
            f = _frame(data, pos, dictionary, dict_id)
        elif 0x184D2A50 <= magic <= 0x184D2A5F:
            st, size = _skippable(data, pos)
            if st:
                return st, result
            pos += size
            f = None
        elif magic == LEGACY_MAGIC:
            f = _legacy(data, pos)
        else:
            return CORRUPTED, result
        if f is not None:
            if f.status == CHECKSUM:
                return CHECKSUM, result + [f.out]
            if f.status:
                return f.status, result
            result.append(f.out)
            pos = f.next
        if pos >= len(data):                                        # :143
            return OK, result
