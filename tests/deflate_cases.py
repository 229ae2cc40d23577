"""A named catalogue of hand-built Deflate streams (tests/deflate_writer.py) that reach the limits of the batch decoders:
15-bit codes and all-ones codes, every length / distance symbol at its extra-bit extremes, distance 32 768, literal runs
around the match record's 8-bit and 15-bit fields, overlapping matches at every residue of an 8-byte word, dense 48-bit
matches at every offset of the warp decoder's 608-bit windows, streams that do not self-synchronise, header edges, stored
block edges and every truncation of the small streams.  Every valid case of families 1, 3 and 4 is also written under an
over-subscribed lit/len, distance and code-length set (family 7), which the batch decoders hand to the generic kernel.

case.data is the unit (start bits in front, trailing junk behind), case.start_bit its first bit, case.expect the intended
output (None: the stream must fail, with status case.status), case.nbits the bits the stream takes (the consumed count).
case.zlib is True when zlib must decode the stream to the same bytes, else the rule under which zlib rejects it."""
import random

from deflate_writer import (DIST_BASE, DIST_EXTRA, LEN_BASE, LEN_EXTRA, DeflateWriter, Match, Raw, as_list, flat,
                            staircase)

OK, TRAP, BAD_STORED, BAD_BTYPE, WRONG_SYMBOL, NOT_FOUND = 0, 2, 101, 102, 103, 104
OVERSUB = "over-subscribed code set: zlib rejects it, the reference keeps the shortest prefix"
RUNS = [255, 256, 257, 511, 32767, 32768, 32769, 65537]
SIXTEEN = bytes(97 + (i & 15) for i in range(256))       # random bytes -> 'a'..'p'


class Case:
    __slots__ = ("name", "family", "data", "start_bit", "nbits", "expect", "status", "zlib", "trace", "stored")

    def __init__(self, name, family, w, expect=True, status=OK, zlib=True, trailing=b"", start_bit=0):
        stream, end = w.finish()
        self.name, self.family = name, family
        self.data = stream + trailing
        self.start_bit = start_bit
        self.nbits = end - start_bit
        self.expect = bytes(w.out) if expect else None
        self.status = status
        self.zlib = zlib if expect else False
        self.trace = w.trace
        self.stored = any(b[0] == "stored" for b in w.trace.blocks)

    @property
    def stream_bytes(self):
        """the bytes that hold the stream (no trailing junk)"""
        return (self.start_bit + self.nbits + 7) // 8


def _w(ov, k, rng):
    return DeflateWriter(oversub=ov, start_bits=k, junk=rng.getrandbits(8) if k else 0)


def _random_prefix(w, rng, n=32768, coded=True):
    """n random bytes the matches can reach back into: a fixed block (no stored block, so the stream may start at any bit)"""
    data = rng.randbytes(n)
    if coded:
        w.fixed([data])
    else:
        for i in range(0, n, 65535):
            w.stored(data[i:i + 65535])


def _phase_literals(lits_by_len, bits):
    """literal tokens whose codes add up to `bits` (lits_by_len: {code length: literal})"""
    out, top = [], max(lits_by_len)
    while bits:
        L = min(bits, top)
        while L not in lits_by_len:
            L -= 1
        out.append(lits_by_len[L])
        bits -= L
    return out


# ------------------------------------------------------------------------------------------------- family 1: code lengths
STAIR_LIT = {
    "len_all_ones": [97, 98, 99, 100, 101, 102, 103, 104, 105, 106, 107, 108, 256, 257, 283, 284],
    "lit_all_ones": [257, 284, 256, 265, 97, 98, 99, 100, 101, 102, 103, 104, 105, 106, 120, 121],
    "eob_all_ones": [97, 284, 98, 257, 99, 270, 100, 101, 102, 103, 104, 105, 106, 107, 255, 256],
}
STAIR_DIST = [3, 4, 5, 10, 15, 20, 25, 26, 27, 0, 1, 2, 6, 7, 28, 29]


def staircase_case(variant, ov, k, rng):
    """lit/len and distance codes of every length 1..15 (a staircase 1, 2, ..., 14, 15, 15), the all-ones 15-bit code of
    each used, every used symbol at its minimum and maximum extra bits, distance 32 768"""
    w = _w(ov, k, rng)
    _random_prefix(w, rng)
    syms = STAIR_LIT[variant]
    lit = as_list(staircase(syms), 286)
    dist = as_list(staircase(STAIR_DIST), 30)
    toks = []
    lens = [s for s in syms if s > 256]
    lits = [s for s in syms if s < 256]
    for rep in range(3):
        for d in STAIR_DIST:
            for ext in (0, (1 << DIST_EXTRA[d]) - 1):
                ls = lens[(d + ext + rep) % len(lens)]
                for lx in (0, (1 << LEN_EXTRA[ls - 257]) - 1):
                    toks += [lits[(d + lx) % len(lits)], lits[-1]]
                    toks.append(Match(LEN_BASE[ls - 257] + lx, DIST_BASE[d] + ext, ls, lx, d, ext))
    w.dynamic(toks, lit, dist, final=True)
    return w


def all_symbols_case(block, ov, k, rng):
    """every length symbol 257..285 and distance symbol 0..29 at its minimum and maximum extra bits, 258 spelled both ways,
    distance 32 768 and distance exactly the output so far"""
    w = _w(ov, k, rng)
    first = bytes(rng.randrange(97, 123) for _ in range(40))
    toks = [first, Match(3, 40), Match(258, 43, 284, 31)]          # a distance equal to the output so far
    w.fixed(toks) if block == "fixed" else w.dynamic(toks)
    _random_prefix(w, rng, 32768 - len(w.out))
    toks = [Match(258, 32768), Match(258, 32768, 284, 31), Match(258, 32768)]   # 32 768 == the output so far, then below it
    for i, ls in enumerate(range(257, 286)):
        for lx in (0, (1 << LEN_EXTRA[ls - 257]) - 1):
            d = (i * 2 + lx) % 30
            for dx in (0, (1 << DIST_EXTRA[d]) - 1):
                toks += [rng.randrange(97, 123), Match(LEN_BASE[ls - 257] + lx, DIST_BASE[d] + dx, ls, lx, d, dx)]
    for d in range(30):
        for dx in (0, (1 << DIST_EXTRA[d]) - 1):
            toks += [rng.randrange(97, 123), Match(3 + d, DIST_BASE[d] + dx, None, None, d, dx)]
    if block == "fixed":
        w.fixed(toks, final=True)
    else:
        lit = as_list(flat(list(range(97, 123)) + [256] + list(range(257, 286))), 286)
        w.dynamic(toks, lit, as_list(flat(range(30)), 30), final=True)
    return w


# Small streams (well under 300 bytes, so the truncation family cuts them at every bit) with 15-bit codes in both alphabets,
# 284 + 31 and wide extra-bit fields: the output grows by 258-byte matches at distance 1, so no random prefix is needed.
COMPACT_LIT = {
    "len_all_ones": [97, 256, 284, 98, 99, 100, 101, 102, 103, 104, 105, 106, 257, 281, 282, 283],   # 283 (5 extra bits)
    "lit_all_ones": [97, 256, 284, 98, 99, 100, 101, 102, 103, 104, 105, 257, 281, 283, 120, 121],   # literal 121
}
COMPACT_DIST = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 16, 17]          # 16/17: 15 bits, 7 extra bits


def compact_long_case(variant, ov, k, rng):
    """a compact stream whose codes reach 15 bits in both alphabets (the all-ones code used in each), with 284 + 31 and
    every distance symbol 0..17 at its minimum and maximum extra bits (up to 7)"""
    w = _w(ov, k, rng)
    syms = COMPACT_LIT[variant]
    lens = [s for s in syms if s > 256]
    lits = [s for s in syms if s < 256]
    toks = [97, Match(258, 1, 284, 31), Match(258, 1, 284, 31)]
    for i, d in enumerate(COMPACT_DIST):
        for ext in (0, (1 << DIST_EXTRA[d]) - 1):
            ls = lens[(i + ext) % len(lens)]
            lx = (1 << LEN_EXTRA[ls - 257]) - 1 if ext else 0
            toks += [lits[(i + ext) % len(lits)], Match(LEN_BASE[ls - 257] + lx, DIST_BASE[d] + ext, ls, lx, d, ext)]
    toks.append(lits[-1])
    w.dynamic(toks, as_list(staircase(syms), 286), as_list(staircase(COMPACT_DIST), 30), final=True)
    return w


def compact_w48_case(ov, k, rng):
    """a compact stream that reaches 24 577 bytes of output through 96 matches of 284 + 31 at distance 1 (a 1-bit length
    code and a 1-bit distance code) and then holds 48-bit matches (15-bit code of 283 + 5 extra bits, 15-bit code of
    distance 29 + 13 extra bits)"""
    w = _w(ov, k, rng)
    lit = staircase([284, 97, 256] + list(range(98, 108)) + [281, 282, 283])
    toks = [97] + [Match(258, 1, 284, 31)] * 96
    for lx, dx in ((0, 0), (31, 191), (17, 64)):
        toks += [rng.randrange(98, 108), Match(195 + lx, 24577 + dx, 283, lx, 29, dx)]
    w.dynamic(toks, as_list(lit, 286), as_list(staircase(W48_DIST), 30), final=True)
    return w


def family1(ov=None):
    rng = random.Random(1001)
    out = []
    for i, v in enumerate(STAIR_LIT):
        out.append((f"stair_{v}", staircase_case(v, ov, i % 8, rng)))
    for i, v in enumerate(COMPACT_LIT):
        out.append((f"compact_{v}", compact_long_case(v, ov, 0, rng)))
    out.append(("compact_w48", compact_w48_case(ov, 0, rng)))
    out.append(("all_symbols_fixed", all_symbols_case("fixed", ov, 3, rng)))
    out.append(("all_symbols_dynamic", all_symbols_case("dynamic", ov, 6, rng)))
    return out


def family1_failing():
    rng = random.Random(1002)
    w = _w(None, 0, rng)
    w.fixed([b"abc", Match(3, 4, unchecked=True)], final=True)
    yield Case("dist_past_output", 1, w, expect=False, status=TRAP)
    w = _w(None, 5, rng)
    _random_prefix(w, rng, 1000)
    w.dynamic([b"xy", Match(258, 1003, 284, 31, unchecked=True)], final=True)
    yield Case("dist_past_output_dynamic", 1, w, expect=False, status=TRAP, start_bit=5)


# ------------------------------------------------------------------------------------------------- family 2: header edges
def family2():
    rng = random.Random(2001)
    az = list(range(97, 123))

    def mk():
        return _w(None, 0, rng)

    # HLIT = 286 (symbol 285 used)
    w = mk()
    w.dynamic([b"abcabc", Match(258, 3)], final=True)
    assert any(s[:2] == ("lit", 285) for s in w.trace.symbols)
    yield Case("hlit_286", 2, w)
    for h in (287, 288):
        w = mk()
        w.dynamic([], as_list(flat(az + [256]), 288), as_list(flat([0, 1]), 2), hlit=h, header_only=True)
        w.bits(0x5A5A, 16)
        yield Case(f"hlit_{h}", 2, w, expect=False, status=WRONG_SYMBOL)
    # HDIST = 32: codes for 30 / 31 present but unused; then used
    dist32 = as_list(flat(range(32)), 32)
    lit = as_list(flat(az + [256, 257, 258, 270]), 286)
    w = mk()
    w.dynamic([b"hellohello", Match(4, 5), b"z", Match(3, 2)], lit, dist32, final=True)
    yield Case("hdist_32_unused", 2, w, zlib="HDIST over 30: zlib rejects the header, the reference reads codes 30/31 as symbols")
    for d in (30, 31):
        w = mk()
        w.dynamic([b"abcdef", Raw(258, 0, d, 0)], lit, dist32, eob=False)
        w.bits(0, 16)
        yield Case(f"hdist_32_uses_{d}", 2, w, expect=False, status=WRONG_SYMBOL)
        w = mk()
        w.fixed([b"abcdef", Raw(258, 0, d, 0)], eob=False)
        w.bits(0, 16)
        yield Case(f"fixed_uses_dist_{d}", 2, w, expect=False, status=WRONG_SYMBOL)
    for s in (286, 287):
        w = mk()
        w.fixed([b"abc", Raw(s)], eob=False)
        w.bits(0, 16)
        yield Case(f"fixed_uses_{s}", 2, w, expect=False, status=WRONG_SYMBOL)
    # HDIST = 1 with length 0, then a length symbol: the distance set is empty
    w = mk()
    w.dynamic([b"abcd", Raw(257)], lit, [0], hdist=1, eob=False)
    w.bits(0xFFFF, 16)
    yield Case("hdist_1_empty_then_match", 2, w, expect=False, status=NOT_FOUND)
    # HCLEN = 4: only 16, 17, 18 and 0 have code-length codes, so every code length is 0
    w = mk()
    w.dynamic([], [0] * 257, [0], hlit=257, hdist=1, hclen=4, cl_lens=as_list({18: 1, 17: 2, 0: 2}, 19),
              cl_ops=[(18, 138), (18, 120)], header_only=True)
    w.bits(0, 24)
    yield Case("hclen_4", 2, w, expect=False, status=NOT_FOUND)
    # HCLEN = 19 where fewer would do (trailing code-length code lengths of 0)
    w = mk()
    w.dynamic([b"ababab", Match(4, 2)], hclen=19, final=True)
    yield Case("hclen_19", 2, w)
    # 7-bit code-length codes
    w = mk()
    w.dynamic([b"abcde", Match(3, 2), b"ea", Match(4, 1), b"abc"],      # code lengths 1..7: eight code-length symbols
              as_list({97: 1, 98: 2, 99: 3, 100: 4, 101: 5, 256: 6, 257: 7, 258: 7}, 286), [1, 1], cl_lens="staircase",
              final=True)
    assert ("cl", 7) in w.trace.lengths
    yield Case("cl_7_bit_codes", 2, w)
    # 16 as the first code-length symbol
    w = mk()
    w.dynamic([], lit, [1, 1], cl_ops=[(16, 3)] + [0] * 10, header_only=True)
    w.bits(0, 16)
    yield Case("cl_16_first", 2, w, expect=False, status=WRONG_SYMBOL)
    # a 16 repeating across the lit/len - distance boundary
    lit5 = as_list(flat(az + [256] + list(range(257, 286)), short_first=False), 286)
    d5 = as_list(flat(range(30), short_first=False), 30)
    w = mk()
    toks = [bytes(rng.randrange(97, 123) for _ in range(300))] + [Match(3 + i, 1 + i * 7) for i in range(40)]
    w.dynamic(toks, lit5, d5, final=True)
    yield Case("cl_16_across_boundary", 2, w)
    # 16 / 17 / 18 that run past the count
    lit_ops = [(18, 97), 6, (16, 6), (16, 6), (16, 6), (16, 4), (16, 3), (18, 133), 6, (16, 6), (16, 6), (16, 6), (16, 6),
               (16, 5)]                                         # 'a'..'z' and 256..285 at 6 bits: 286 lit/len lengths
    assert sum(1 if isinstance(o, int) else o[1] for o in lit_ops) == 286
    for name, tail in (("cl_16_overshoots", [2, 2, 2, 2, (16, 6), (16, 6)]), ("cl_17_overshoots", [2, 2, 2, 2, (17, 10)]),
                       ("cl_18_overshoots", [2, 2, 2, 2, (18, 20)])):
        w = mk()
        w.dynamic([], [0] * 286, [0] * 12, hlit=286, hdist=12, cl_ops=lit_ops + tail, header_only=True)
        w.bits(0, 16)
        yield Case(name, 2, w, expect=False, status=WRONG_SYMBOL)
    # no end-of-block code
    w = mk()
    w.dynamic([bytes(rng.randrange(97, 123) for _ in range(50))], as_list(flat(az), 286), [1, 1], eob=False)
    w.bits(0, 5)
    yield Case("no_eob_code", 2, w, expect=False, status=NOT_FOUND)
    # an empty dynamic block (end of block only), then a fixed block
    w = mk()
    w.dynamic([], as_list({256: 1}, 257), [0], hdist=1)
    w.fixed([b"after"], final=True)
    yield Case("empty_dynamic_block", 2, w)


# ------------------------------------------------------------------------------------------------- family 3: records
def run_case(n, how, ov, k, rng):
    """a literal run of n bytes, then a match; a few literals; another run of up to 511 bytes (made of the same block
    kind), then a far match"""
    w = _w(ov, k, rng)
    data = rng.randbytes(n).translate(SIXTEEN)

    def put_run(data, last_toks, final=False):
        if how == "stored":
            for i in range(0, len(data), 65535):
                w.stored(data[i:i + 65535])
            w.fixed(last_toks, final=final)
        elif how == "fixed":
            w.fixed([data] + last_toks, final=final)
        elif how == "dynamic":
            w.dynamic([data] + last_toks, final=final)
        else:                                   # stored, then fixed, then dynamic pieces of the one run
            a, b = len(data) // 3, 2 * len(data) // 3
            for i in range(0, a, 65535):
                w.stored(data[i:min(a, i + 65535)])
            w.fixed([data[a:b]])
            w.dynamic([data[b:]] + last_toks, final=final)

    put_run(data, [Match(10, min(n, 300)), 120, 121, 122])
    put_run(data[:-512:-1], [Match(258, min(len(w.out), 32768)), Match(3, 1)], final=True)
    return w


def overlap_case(r, ov, k, rng):
    """overlapping matches, distances 1..8 x lengths 3..10 and 258, each starting at output residue r mod 8"""
    w = _w(ov, k, rng)
    toks, n = [bytes(rng.randrange(97, 123) for _ in range(16))], 16
    for d in range(1, 9):
        for ln in list(range(3, 11)) + [258]:
            pad = (r - n) % 8
            toks.append(bytes(rng.randrange(97, 123) for _ in range(pad)))
            toks.append(Match(ln, d))
            n += pad + ln
    w.fixed(toks, final=True)
    return w


def near_far_case(seed, ov, k, rng):
    """chains of near matches (distance 1..16) mixed with far ones"""
    w = _w(ov, k, rng)
    _random_prefix(w, rng)
    r = random.Random(seed)
    toks, n = [], len(w.out)
    for _ in range(1500):
        x = r.random()
        if x < 0.55:
            m = Match(r.randrange(3, 41), r.randrange(1, 17))
        elif x < 0.75:
            m = Match(r.choice([3, 4, 258, r.randrange(3, 259)]), r.randrange(16384, 32769))
        else:
            m = None
            lit = bytes(r.randrange(97, 123) for _ in range(r.randrange(0, 6)))
            toks.append(lit)
            n += len(lit)
        if m is not None:
            toks.append(m)
            n += m.length
    w.dynamic(toks, final=True)
    return w


def family3(ov=None):
    rng = random.Random(3001)
    out = []
    for i, n in enumerate(RUNS):
        for j, how in enumerate(("stored", "fixed", "dynamic", "mixed")):
            k = 0 if how in ("stored", "mixed") else (i + j) % 8
            out.append((f"run_{n}_{how}", run_case(n, how, ov, k, rng)))
    for r in range(8):
        out.append((f"overlap_residue_{r}", overlap_case(r, ov, r, rng)))
    for s in range(3):
        out.append((f"near_far_{s}", near_far_case(3100 + s, ov, s + 2, rng)))
    return out


# ------------------------------------------------------------------------------------------------- family 4: K1w windows
W48_LIT = [65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 75, 76, 77, 256, 283, 284]   # 'A'..'M' 1..13 bits, EOB 14, 283/284 15
W48_DIST = list(range(14)) + [28, 29]                                          # 0..13 1..14 bits, 28/29 15 bits
W48_LONG = (0, 17, 40)                                                         # phases whose run crosses a chunk end


def w48_case(phase, ov, k, rng):
    """`phase` bits of literals, then a dense run of 48-bit matches (15-bit code of 284 + 5 extra bits, 15-bit code of
    distance 29 + 13 extra bits)"""
    w = _w(ov, k, rng)
    _random_prefix(w, rng)
    lit = staircase(W48_LIT)
    toks = _phase_literals({L: s for s, L in lit.items() if s < 256}, phase)
    for _ in range(420 if phase in W48_LONG else 40):
        lx, dx = rng.randrange(32), rng.randrange(1 << 13)
        toks.append(Match(227 + lx, 24577 + dx, 284, lx, 29, dx))
    w.dynamic(toks, as_list(lit, 286), as_list(staircase(W48_DIST), 30), final=True)
    return w


def nosync_case(ov, k, rng):
    """255 literal codes of 8 bits (0..254; 255 and end of block at 9): nearly every bit offset parses as a run of
    literals, so wrongly guessed window starts do not fall into step with the true chain.  A 9-bit literal every 50 moves
    the true chain off the 8-bit grid of the guessed starts (a window is 76 bytes of 8 bits)."""
    w = _w(ov, k, rng)
    lit = {s: 8 for s in range(255)}
    lit.update({255: 9, 256: 9})
    body = rng.randbytes(9000).replace(b"\xff", b"\x00")
    w.dynamic([b"\xff".join(body[i:i + 50] for i in range(0, len(body), 50))], as_list(lit, 286), [1, 1], final=True)
    return w


def hazard_cases(ov, rng):
    """streams whose misaligned parses run into end of block, 286/287, distance codes 30/31 or distances past the output"""
    out = []
    w = _w(ov, 1, rng)
    toks = [bytes(rng.getrandbits(8) for _ in range(64))]
    for _ in range(700):
        toks.append(bytes(rng.getrandbits(8) for _ in range(rng.randrange(1, 12))))
        toks.append(Match(rng.randrange(3, 30), rng.randrange(1, 60)))
    w.fixed(toks, final=True)
    out.append(("hazard_fixed_286_287", w))
    w = _w(ov, 2, rng)
    az = list(range(97, 123))
    lit = {256: 2, 97: 2, 98: 2}
    lit.update({s: L + 2 for s, L in flat(az[2:]).items()})
    w.dynamic([bytes(rng.choice(az) for _ in range(7000))], as_list(lit, 286), [1, 1], final=True)
    out.append(("hazard_short_eob", w))
    w = _w(ov, 3, rng)
    toks = [b"ab"]
    for i in range(2500):
        toks.append(Match(rng.randrange(3, 11), rng.randrange(1, 3)))
        if i % 7 == 0:
            toks.append(rng.randrange(97, 100))
    w.fixed(toks, final=True)
    out.append(("hazard_near_start", w))
    return out


def hazard_dist3031(rng):
    w = _w(None, 4, rng)
    toks = [bytes(rng.randrange(256) for _ in range(100))]
    for _ in range(800):
        toks.append(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 10))))
        toks.append(Match(rng.randrange(3, 11), rng.randrange(1, 100)))
    w.dynamic(toks, as_list(flat(list(range(256)) + [256] + list(range(257, 265))), 286), as_list(flat(range(32)), 32), final=True)
    return w


def family4(ov=None):
    rng = random.Random(4001)
    out = [(f"w48_phase_{p}", w48_case(p, ov, p % 8, rng)) for p in range(48)]
    out.append(("nosync_8bit", nosync_case(ov, 5, rng)))
    out += hazard_cases(ov, rng)
    return out


# ------------------------------------------------------------------------------------------------- family 5: blocks, stored
def family5():
    rng = random.Random(5001)
    w = _w(None, 0, rng)
    for i in range(2000):
        lits = bytes(rng.randrange(97, 123) for _ in range(rng.randrange(1, 4)))
        toks = [lits] + ([Match(3, rng.randrange(1, len(w.out) + len(lits) + 1))] if i % 3 and i > 3 else [])
        if i % 3 == 0:
            w.stored(lits, final=i == 1999)
        elif i % 3 == 1:
            w.fixed(toks, final=i == 1999)
        else:
            w.dynamic(toks, final=i == 1999)
    yield Case("tiny_blocks_2000", 5, w)
    for n in (0, 65535):
        w = _w(None, 0, rng)
        w.stored(rng.randbytes(n), final=True)
        yield Case(f"stored_len_{n}", 5, w)
    for ln, nln in ((5, 0), (0xF0, 0x0F00), (0, 0)):
        w = _w(None, 0, rng)
        w.stored(bytes(rng.getrandbits(8) for _ in range(ln)), length=ln, nlength=nln)
        w.fixed([b"ok"], final=True)
        yield Case(f"stored_and_zero_{ln:x}_{nln:x}", 5, w,
                   zlib="LEN and NLEN are checked by AND in the reference, as complements in zlib")
    w = _w(None, 0, rng)
    w.stored(b"hello", length=5, nlength=5, final=True)
    yield Case("stored_and_nonzero", 5, w, expect=False, status=BAD_STORED)
    w = _w(None, 0, rng)
    w.stored(bytes(50), length=100, final=True)
    yield Case("stored_len_past_end", 5, w, expect=False, status=BAD_STORED)
    for p in range(8):
        w = _w(None, 0, rng)
        w.fixed([97, 98] + [200] * ((p - 2) % 8))                  # 3 + 2 x 8 + 9 b + 7 bits: the next block starts at bit p
        assert w.w.pos % 8 == p
        w.stored(bytes(rng.getrandbits(8) for _ in range(20)), final=True)
        yield Case(f"stored_at_phase_{p}", 5, w)


# ------------------------------------------------------------------------------------------------- family 6: ends of input
def family6_whole():
    rng = random.Random(6001)
    w = _w(None, 0, rng)
    w.fixed([97, 98, 99] + [200] * 6, final=True)                 # 3 + 3 x 8 + 6 x 9 + 7 = 88 bits
    assert w.w.pos % 8 == 0
    yield Case("eob_on_last_bit", 6, w, trailing=b"")


class Cut:
    """One truncation unit: `data` is the stream (shifted by `start_bit`) cut after `avail` of its bits' bytes, `tail` the
    rest of that stream, which lies behind the unit in memory so that a decoder reading past its end sees the true
    continuation; `case` is the case it was cut from."""
    __slots__ = ("name", "data", "start_bit", "tail", "avail", "case")

    def __init__(self, name, data, start_bit, tail, case):
        self.name, self.data, self.start_bit, self.tail, self.case = name, data, start_bit, tail, case
        self.avail = 8 * len(data) - start_bit           # stream bits the unit holds


def truncations(cases, limit=300):
    """every valid compact case (under `limit` bytes) cut at every byte, and (when it holds no stored block, whose length
    field would move) shifted by start bits 1..7 and cut, so that a unit ends at every bit of the stream.  The first byte
    stays when there are start bits (they lie inside it).  -> [Cut]"""
    out = []
    rng = random.Random(6002)
    for c in cases:
        if c.expect is None or c.stream_bytes > limit or (c.stored and c.start_bit):
            continue
        v = int.from_bytes(c.data[:c.stream_bytes], "little") >> c.start_bit
        for k in range(8):
            if k and c.stored:
                continue
            data = ((v << k) | rng.getrandbits(k)).to_bytes((k + c.nbits + 7) // 8, "little")
            for cut in range(1 if k else 0, len(data)):
                out.append(Cut(f"{c.name}/k{k}/cut{cut}", data[:cut], k, data[cut:], c))
    return out


# ------------------------------------------------------------------------------------------------- the catalogue
def _valid(fam, items, ov):
    """Cases from (name, writer) pairs; every other one is followed by trailing junk"""
    return [Case(name + (f"/over_{ov}" if ov else ""), 7 if ov else fam, w, zlib=OVERSUB if ov else True,
                 trailing=bytes([0x5A, 0xC3, 0x00]) if i % 2 else b"", start_bit=w.trace.start_bits)
            for i, (name, w) in enumerate(items)]


_CACHE = {}


def catalogue():
    """every case (truncations not included) -> [Case]"""
    if "all" in _CACHE:
        return _CACHE["all"]
    cases = []
    for fam, make in ((1, family1), (3, family3), (4, family4)):
        cases += _valid(fam, make(), None)
        for ov in ("lit", "dist", "cl"):
            cases += _valid(fam, make(ov), ov)
    cases += list(family1_failing())
    cases += list(family2())
    rng = random.Random(4002)
    cases += _valid(4, [("hazard_dist_30_31", hazard_dist3031(rng))], None)
    cases[-1].zlib = "HDIST over 30: zlib rejects the header, the reference reads codes 30/31 as symbols"
    cases += list(family5())
    cases += list(family6_whole())
    names = [c.name for c in cases]
    assert len(set(names)) == len(names)
    _CACHE["all"] = cases
    return cases


def truncation_units():
    if "trunc" not in _CACHE:
        _CACHE["trunc"] = truncations(catalogue())
    return _CACHE["trunc"]
