"""Deflate streams that decode to 2 GiB and more, up to and just past the largest output a Deflate unit may have
(OUT_MAX = 0xFFFFFFF0 bytes, inflate.cuh).  Each is one dynamic block, built from byte arithmetic rather than a token
loop, whose output is periodic: output[p] = SEED[p % P], P = 251.  P is coprime with 16, so a 16-byte chunk stored at
the wrong address, or a byte left unwritten, differs from the pattern wherever it lands.

A stream is
    SEED as P literals; HEAD near matches (258 at distance P) -> more than FAR bytes of output;
    the bulk: 258-byte matches at distance FAR = 8 P, each the same 11 bits (lit/len 285 has a 1-bit code and the
      distance code a 1-bit code), so the bulk is a run of identical 11-byte groups after the first;
    a near tail: 258-byte matches at distance P (one or two shorter ones to land on the length), at least RING bytes of
      them, so that lz_resolve_kernel reads their sources from its ring right up to the end of the output;
    the end: a match (`tail="match"`), a literal run (`"literal"`) or the end of the block and a final stored block
      (`"stored"`), of `tail_len` bytes.
The far bulk keeps lz_resolve_kernel fast (its matches replay 16 at a time); the near head and tail cover the chained
replay and, at the ceiling, the far/near test on source positions above 2^32 - RING."""
import zlib
from dataclasses import dataclass

import numpy as np

import deflate_writer as W

P = 251
SEED = bytes((37 * i + 11) % 256 for i in range(P))
FAR = 8 * P                     # > RING - 258: lz_resolve_kernel replays these matches from the output it has flushed
HEAD = 8                        # near matches before the bulk: P + 8 * 258 > FAR
NEAR_TAIL = 2304                # near-match bytes before the end (> RING = 2048)
OUT_MAX = 0xFFFFFFF0
GIB = 1 << 30


def _lit_lengths():
    """285 gets a 1-bit code; every other lit/len symbol (literals, end of block, lengths 257-284) a flat code in the
    other half, so every byte value and every length can be written"""
    rest = W.flat([s for s in range(286) if s != 285])
    lens = {s: L + 1 for s, L in rest.items()}
    lens[285] = 1
    assert W.kraft(lens) == 1
    return W.as_list(lens, 286)


LIT_LENS = _lit_lengths()
DSYM_NEAR, DEXTRA_NEAR = W.dist_symbol(P)
DSYM_FAR, DEXTRA_FAR = W.dist_symbol(FAR)
DIST_LENS = W.as_list({DSYM_NEAR: 1, DSYM_FAR: 1}, 30)
LIT = W.Code(LIT_LENS)
DIST = W.Code(DIST_LENS)


def expected(p0, n):
    """output bytes [p0, p0 + n) of every case"""
    k = p0 % P
    reps = (k + n + P - 1) // P
    return np.frombuffer(SEED * reps, dtype=np.uint8)[k:k + n]


@dataclass
class Case:
    name: str
    data: bytes                 # the raw Deflate stream
    size: int                   # its output length
    tail: str
    tail_len: int
    nbits: int                  # bits the decoder consumes: up to the end of the final block

    @property
    def decodes(self):
        return self.size <= OUT_MAX


class _Stream:
    """a BitWriter plus the output length so far"""

    def __init__(self):
        self.w = W.BitWriter()
        self.n = 0

    def lit(self, b):
        self.w.code(LIT.codes[b], LIT_LENS[b])
        self.n += 1

    def literals(self, count):
        for b in expected(self.n, count):
            self.lit(int(b))

    def match(self, length, dist):
        lsym, lextra = W.len_symbol(length)
        dsym, dextra = W.dist_symbol(dist)
        assert dist <= self.n and DIST_LENS[dsym]
        self.w.code(LIT.codes[lsym], LIT_LENS[lsym])
        self.w.bits(lextra, W.LEN_EXTRA[lsym - 257])
        self.w.code(DIST.codes[dsym], DIST_LENS[dsym])
        self.w.bits(dextra, W.DIST_EXTRA[dsym])
        self.n += length

    def far_bulk(self, count):
        """`count` 258-byte matches at distance FAR: eight of them are 88 bits, so after the first group of eight every
        group adds the same 11 bytes to the stream"""
        groups, rest = divmod(count, 8)
        if groups >= 2:
            for _ in range(8):
                self.match(258, FAR)
            before = len(self.w.out)
            for _ in range(8):
                self.match(258, FAR)
            unit = bytes(self.w.out[before:])
            assert len(unit) == 11
            self.w.out += unit * (groups - 2)
            self.w.pos += 88 * (groups - 2)
            self.n += 8 * 258 * (groups - 2)
        else:
            rest += 8 * groups
        for _ in range(rest):
            self.match(258, FAR)

    def near(self, nbytes):
        """matches at distance P covering exactly `nbytes` (>= 3) bytes"""
        full, r = divmod(nbytes, 258)
        if r in (1, 2):                      # 258 + r as two matches
            full -= 1
            parts = [258] * full + [129, 129 + r]
        else:
            parts = [258] * full + ([r] if r else [])
        for ln in parts:
            self.match(ln, P)


def build(size, tail="match", tail_len=None, name=None):
    """a stream that decodes to `size` bytes and ends as `tail` says (`tail_len` bytes of literals or stored data; the
    match tail ends with a match)"""
    assert tail in ("match", "literal", "stored")
    if tail_len is None:
        tail_len = {"match": 0, "literal": 24, "stored": 1000}[tail]
    s = _Stream()
    s.w.bits(1 if tail != "stored" else 0, 1)          # BFINAL
    s.w.bits(2, 2)
    hlit = 286
    hdist = max(i + 1 for i, L in enumerate(DIST_LENS) if L)
    lens = LIT_LENS[:hlit] + DIST_LENS[:hdist]
    ops = W.rle(lens)
    freq = {}
    for op in ops:
        k = op if isinstance(op, int) else op[0]
        freq[k] = freq.get(k, 0) + 1
    cl_lens = W.as_list(W.flat(sorted(freq)), 19)
    hclen = max(4, max(i + 1 for i, k in enumerate(W.CL_ORDER) if cl_lens[k]))
    s.w.bits(hlit - 257, 5)
    s.w.bits(hdist - 1, 5)
    s.w.bits(hclen - 4, 4)
    for i in range(hclen):
        s.w.bits(cl_lens[W.CL_ORDER[i]], 3)
    clc = W.Code([cl_lens[k] if W.CL_ORDER.index(k) < hclen else 0 for k in range(19)])
    for op in ops:
        k, reps = (op, None) if isinstance(op, int) else op
        s.w.code(clc.codes[k], cl_lens[k])
        if k in (16, 17, 18):
            s.w.bits(reps - {16: 3, 17: 3, 18: 11}[k], {16: 2, 17: 3, 18: 7}[k])
    s.literals(P)
    for _ in range(HEAD):
        s.match(258, P)
    end_tail = 0 if tail == "match" else tail_len
    body = size - s.n - end_tail                       # far bulk + near tail
    assert body >= NEAR_TAIL + 258, "too small for the layout"
    nbulk = (body - NEAR_TAIL) // 258
    s.far_bulk(nbulk)
    s.near(size - end_tail - s.n)
    if tail == "literal":
        s.literals(tail_len)
    s.w.code(LIT.codes[256], LIT_LENS[256])
    if tail == "stored":
        assert tail_len <= 0xFFFF
        s.w.bits(1, 1)
        s.w.bits(0, 2)
        s.w.align()
        s.w.bits(tail_len, 16)
        s.w.bits(~tail_len & 0xFFFF, 16)
        s.w.out += expected(s.n, tail_len).tobytes()
        s.w.pos += 8 * tail_len
        s.n += tail_len
    assert s.n == size
    return Case(name or f"{size:#x}-{tail}", s.w.data(), size, tail, tail_len, s.w.pos)


# ------------------------------------------------------------------------------------------------ the catalogue
def crossing():
    """2^31 + 1, ending on a match: the flush that crosses 2^31"""
    return build((1 << 31) + 1, "match", name="2^31+1")


def ceiling():
    """exactly OUT_MAX, ending on a match"""
    return build(OUT_MAX, "match", name="ceiling")


def lengths():
    """every size that must decode, one case each (the crossing and ceiling cases included)"""
    out = [build((1 << 31) - 1, "match", name="2^31-1"), build(1 << 31, "literal", name="2^31"), crossing(),
           build(3 * GIB, "stored", name="3GiB-stored"), ceiling()]
    for k, tail in ((1, "literal"), (5, "stored"), (11, "match"), (15, "literal"), (16, "match")):
        out.append(build(OUT_MAX - k, tail, name=f"ceiling-{k}-{tail}"))
    out.append(build(OUT_MAX - 3, "literal", tail_len=1, name="ceiling-3-one-literal"))
    out.append(build(OUT_MAX, "stored", tail_len=0xFFFF, name="ceiling-stored-64k"))
    return out


def past_ceiling():
    """units that would decode to more than OUT_MAX bytes: one more byte by a match, by one literal, 2^32 by sixteen
    literals, and a stored block that crosses both OUT_MAX and 2^32"""
    return [build(OUT_MAX + 1, "match", name="over-by-match"),
            build(OUT_MAX + 1, "literal", tail_len=1, name="over-by-1-literal"),
            build(OUT_MAX + 16, "literal", tail_len=16, name="over-by-16-literals"),
            build(OUT_MAX + 500, "stored", tail_len=1000, name="over-by-stored")]


def small():
    """a 1 MiB case of the same layout, for quick checks of the builder"""
    return build(1 << 20, "literal", name="1MiB")


def zlib_check(size, tail, tail_len):
    """builds the case and decodes it with zlib in slices -> (output length, the stream ended cleanly with its final
    block, the first output position that differs from the pattern or None)"""
    data = build(size, tail, tail_len).data
    slice_bytes = 64 << 20
    tiled = SEED * ((slice_bytes + 2 * P) // P)
    d = zlib.decompressobj(-15)
    n, pos, bad = 0, 0, None
    while not d.eof:
        chunk = d.unconsumed_tail
        if not chunk:
            chunk = data[pos:pos + (1 << 20)]
            pos += len(chunk)
        out = d.decompress(chunk, slice_bytes)
        if not out and not chunk:
            break
        k = n % P
        if bad is None and out != tiled[k:k + len(out)]:
            a = np.frombuffer(out, dtype=np.uint8)
            bad = n + int(np.flatnonzero(a != expected(n, len(out)))[0])
        n += len(out)
    return n, d.eof and not d.unused_data and pos >= len(data), bad
