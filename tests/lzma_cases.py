"""A named catalogue of hand-built LZMA and LZMA2 streams (written by tests/lzma_writer.py) and every byte cut of its small
ones.  Each case carries the reference's answer from the writer's model of the Swift decoder; `batch` is what the batched
entry points answer where they may differ (DESIGN §6: UNSUPPORTED for lc + lp > 4, and for raw properties no properties
byte can express, which the oracle and the single-stream API refuse too)."""
import random

import lzma_writer as W
from lzma_writer import SHORT, end, lit, lit_vs_match, match, rep

MIB = 1 << 20


class Case:
    """form "raw" (LZMA.decompress(data:properties:uncompressedSize:)), "alone" (.lzma header, LZMA.decompress(data:)) or
    "lzma2" (LZMA2 chunks, the dictionary byte apart).  `liblzma`: liblzma's raw decoder takes it and must agree."""

    def __init__(self, name, family, form, data, lc=3, lp=0, pb=2, dict_size=1 << 16, usize=-1, dict_byte=None, liblzma=False):
        self.name, self.family, self.form, self.data = name, family, form, bytes(data)
        self.lc, self.lp, self.pb, self.dict_size, self.usize, self.dict_byte = lc, lp, pb, dict_size, usize, dict_byte
        if form == "raw":
            self.model = W.decode_lzma(self.data, lc, lp, pb, dict_size, usize)
        elif form == "alone":
            self.model = W.decode_lzma_alone(self.data)
        else:
            self.model = W.decode_lzma2(self.data, dict_byte)
        self.liblzma = liblzma and self.model.status == W.OK
        # no properties byte holds these: the oracle and the engine refuse them (the model keeps the reference's answer)
        self.unexpressible = form == "raw" and not (0 <= lc <= 8 and 0 <= lp <= 4 and 0 <= pb <= 4)

    @property
    def status(self):
        """the oracle's and the single-stream API's answer"""
        return W.UNSUPPORTED if self.unexpressible else self.model.status

    @property
    def batch(self):
        return W.UNSUPPORTED if self.unexpressible else self.model.batch_status()

    @property
    def props(self):
        return self.lc | self.lp << 8 | self.pb << 16


def raw(name, family, ops, lc=3, lp=0, pb=2, dict_size=1 << 16, known=True, usize=None, extra=0, first=None, liblzma=True):
    """a raw LZMA case; `known`: the size is given (the true one unless `usize`), else -1 (the stream needs its end marker)"""
    data = W.write_lzma(ops, lc, lp, pb, dict_size, extra, first)
    if usize is None:
        m = W.Model(lc, lp, pb, dict_size)
        m.reset()
        W.encode_ops(m, [o for o in ops if not (o[0] == "match" and o[2] == W.END_MARKER)])
        usize = len(m.out) if known else -1
    ok_props = lc + lp <= 4 and 0 <= lc and 0 <= lp and 0 <= pb <= 4 and 4096 <= dict_size < 1 << 32
    return Case(name, family, "raw", data, lc, lp, pb, dict_size, usize, liblzma=liblzma and ok_props)


def lzma2(name, family, chunks, dict_byte=18, end_byte=True, liblzma=False):
    ds = W.lzma2_dict_size(dict_byte) or 4096
    return Case(name, family, "lzma2", W.write_lzma2(chunks, ds, end_byte), dict_byte=dict_byte, liblzma=liblzma)


def text(n, seed):
    rng = random.Random(seed)
    words = [b"lzma", b"range", b"coder", b"literal", b"match", b" ", b"rep", b"\n", b"state", b"dict"]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words)
    return bytes(out[:n])


def lits(bs):
    return [lit(b) for b in bs]


def mixed_ops(seed, n=64):
    """literals over every low bit pattern, then each symbol kind once: a stream every properties byte can decode"""
    t = text(n, seed)
    return (lits(b"\xFF" * 40 + t) + [match(5, 3), rep(1, 4), SHORT, lit(1), match(273, 30), rep(3, 2), rep(2, 9),
                                      lit_vs_match(3), rep(0, 17)] + lits(bytes(range(0, 256, 7))))


# ---------------------------------------------------------------------------------------------------------- families
def properties():
    """every properties byte in .lzma headers (known size and end marker), the refused bytes 225-255, and raw lc 9 / pb 5"""
    out = []
    for b in range(225):
        lc, lp, pb = b % 9, (b // 9) % 5, b // 45
        ops = mixed_ops(b)
        for known in (True, False):
            m = W.Model(lc, lp, pb, 1 << 16)
            m.reset()
            W.encode_ops(m, ops)
            body = W.write_lzma(ops + ([] if known else [end()]), lc, lp, pb, 1 << 16)
            head = W.lzma_header(b, 1 << 16, len(m.out) if known else -1)
            out.append(Case(f"props_{b}_{'known' if known else 'marker'}", 1, "alone", head + body))
    for b in range(225, 256):
        out.append(Case(f"props_{b}_refused", 1, "alone", W.lzma_header(b, 1 << 16, 4) + W.write_lzma(lits(b"abcd"))))
    # raw properties past a properties byte: what the reference does with them (the engine refuses them all)
    out.append(raw("raw_lc9_decodes", 1, mixed_ops(900) + [end()], lc=9, known=False))
    out.append(raw("raw_lc9_lp4", 1, lits(b"\xFF" * 20 + text(80, 901)) + [end()], lc=9, lp=4, known=False))
    out.append(raw("raw_pb5_literals_decode", 1, lits(text(100, 902)) + [end(2)], pb=5, known=True))
    out.append(raw("raw_pb5_match_at_posstate_17", 1, lits(text(17, 903)) + [match(4, 2)] + lits(b"zz"), pb=5))
    out.append(raw("raw_pb5_match_at_posstate_3", 1, lits(text(3, 904)) + [match(4, 2)] + lits(b"zz"), pb=5))
    out.append(raw("raw_lp5", 1, lits(text(40, 905)), lp=5))
    return out


DICTS = [0, 1, 2, 4095, 4096, (1 << 32) - 1, -1]


def dictionaries():
    out = []
    for ds in DICTS:
        n = 5000 if 0 < ds <= 4096 else 300
        t = text(n, 1000 + (ds & 0xFFFF))
        tag = "m1" if ds < 0 else str(ds)
        out.append(raw(f"dict_{tag}_literals", 2, lits(t), dict_size=ds))
        out.append(raw(f"dict_{tag}_rep0_after_literals", 2, lits(t[:50]) + [rep(0, 5)] + lits(b"ab"), dict_size=ds))
        out.append(raw(f"dict_{tag}_short_rep", 2, lits(t[:50]) + [SHORT, lit(9)], dict_size=ds))
        if ds >= 1:
            for d, what in ((ds - 1, "size_minus_1"), (ds, "size")):
                if d < 1 << 20:
                    out.append(raw(f"dict_{tag}_match_at_{what}", 2, lits(t) + [match(3, d)] + lits(b"xy"), dict_size=ds))
        # rep0 == dictEnd < dictSize: accepted by the range check, then byte(at:) takes its wrapped branch
        out.append(raw(f"dict_{tag}_match_at_dict_end", 2, lits(t[:3]) + [match(2, 3)], dict_size=ds))
        if 0 <= ds < 1 << 32:                # the header form: nothing clamps the size
            m = W.Model(3, 0, 2, ds)
            m.reset()
            W.encode_ops(m, lits(t[:300]))
            out.append(Case(f"dict_{tag}_header", 2, "alone", W.lzma_header(93, ds, len(m.out)) + W.write_lzma(lits(t[:300]), dict_size=ds)))
    return out


def slot_base(s):
    return s if s < 4 else (2 | (s & 1)) << ((s >> 1) - 1)


def pos_slots():
    out = []
    t = text(300, 2000)
    # every reverse-tree value of slots 4..13 and every align value (slot 14, direct bits 0..3)
    ops = lits(t)
    for s in range(4, 14):
        for r in range(1 << ((s >> 1) - 1)):
            ops.append(match(2 + r % 5, slot_base(s) + r))
    for r in range(64):
        ops.append(match(3, 128 + r))
    out.append(raw("slots_4_to_13_every_value_and_align", 3, ops + [end()], known=False))
    # slots 0..45 as real matches in an output grown to 8 MiB by 273-byte reps
    ops = lits(t) + [match(273, 299)] + [rep(0, 273)] * (8 * MIB // 273)
    for s in range(46):
        ops.append(match(2 + s % 7, slot_base(s) + (0 if s < 4 else 1 << ((s >> 1) - 2))))
    out.append(raw("slots_0_to_45_in_8_mib", 3, ops, dict_size=1 << 24, liblzma=True))
    for s in range(46, 64):
        out.append(raw(f"slot_{s}_not_enough", 3, lits(t[:20]) + [match(2, slot_base(s))], dict_size=1 << 24))
    out.append(raw("slot_63_all_but_one", 3, lits(t[:20]) + [match(2, W.END_MARKER - 1)], dict_size=1 << 24))
    out.append(raw("slot_63_end_marker", 3, lits(t[:20]) + [end()], known=False))
    return out


def lengths():
    """lengths 2..273 through each length coder at every posState, pb = 4"""
    out = []
    for coder in ("match", "rep"):
        need = {(L, ps) for L in range(2, 274) for ps in range(16)}
        ops, pos = lits(text(64, 3000)), 64
        while need:
            ps = pos % 16
            L = next((L for L in range(2, 274) if (L, ps) in need), None)
            if L is None:
                ops.append(lit(pos & 0xFF))
                pos += 1
                continue
            need.discard((L, ps))
            ops.append(match(L, 0) if coder == "match" else rep(1, L))   # (rep0 at state 11 / posState 15 traps)
            pos += L
        out.append(raw(f"lengths_{coder}_every_posstate_pb4", 4, ops, pb=4, dict_size=1 << 22))
    return out


# the shortest path from state 0 to each state
STATE_PATHS = {0: [], 7: [match(2, 0)], 8: [rep(1, 2)], 9: [SHORT], 10: [match(2, 0), match(2, 1)], 11: [match(2, 0), rep(0, 2)],
               4: [match(2, 0), lit(1)], 5: [rep(1, 2), lit(1)], 6: [SHORT, lit(1)], 1: [match(2, 0), lit(1), lit(2)],
               2: [rep(1, 2), lit(1), lit(2)], 3: [SHORT, lit(1), lit(2)]}
KINDS = {"lit": [lit(0x41)], "match": [match(3, 2)], "rep0": [rep(0, 3)], "rep1": [rep(1, 3)], "rep2": [rep(2, 3)],
         "rep3": [rep(3, 3)], "short": [SHORT], "end": []}


def states():
    out = []
    for s, path in STATE_PATHS.items():
        for k, op in KINDS.items():
            out.append(raw(f"state_{s}_{k}", 5, lits(text(16, 4000 + s)) + path + op + [end()], known=False))
    # isRep0Long at state 11 / posState 15 with pb = 4 is entry 432 of 432: a short rep and a long rep0 both trap; 431 does not
    for ps in (14, 15):
        for k, op in (("short", SHORT), ("rep0", rep(0, 2))):
            pre = lits(text(16 + (ps - 4) % 16, 4100))        # 16 + x literals, then 2 + 2 bytes of match and rep: x + 4 = ps
            out.append(raw(f"state_11_posstate_{ps}_{k}", 5, pre + [match(2, 0), rep(0, 2), op, end()], pb=4, known=False))
    # matched literals leaving the match byte at each bit, and following it to the end
    ops = lits(text(40, 4200))
    for k in list(range(8)) + [None]:
        ops += [match(2, 7), lit_vs_match(k), match(3, 11), lit_vs_match(k)]
    out.append(raw("matched_literal_every_bit", 5, ops + [end()], known=False))
    return out


def termination():
    out = []
    t = text(40, 5000)
    n = len(t)
    for k, op in (("literal", lit(1)), ("rep", rep(0, 2)), ("short", SHORT), ("match", match(2, 3)), ("end", end())):
        out.append(raw(f"size_reached_then_{k}", 6, lits(t) + [op], usize=n))
    out.append(raw("size_reached_code_zero", 6, lits(t), usize=n))
    out.append(raw("size_reached_code_nonzero", 6, lits(t), usize=n, extra=1))
    out.append(raw("size_reached_code_nonzero_more_bytes", 6, lits(t), usize=n, extra=0x10000))
    out.append(raw("end_marker_before_size", 6, lits(t) + [end()], usize=n + 5))
    out.append(raw("end_marker_then_literal", 6, lits(t) + [end(), lit(5)], known=False))
    out.append(raw("end_marker_then_match", 6, lits(t) + [end(), match(2, 1), end()], known=False))
    out.append(raw("end_marker_code_nonzero", 6, lits(t) + [end()], known=False, extra=3))
    out.append(raw("end_marker_length_273", 6, lits(t) + [end(273)], known=False))
    out.append(raw("match_longer_than_left", 6, lits(t) + [match(10, 3)], usize=n + 9))
    out.append(raw("rep_longer_than_left", 6, lits(t) + [rep(0, 3)], usize=n + 2))
    out.append(raw("first_byte_1", 6, lits(t), first=1))
    out.append(raw("first_byte_ff", 6, lits(t), first=0xFF))
    out.append(raw("size_zero_empty", 6, [], usize=0))
    out.append(raw("size_zero_then_literal", 6, [lit(3)], usize=0))
    for k in range(5):
        out.append(Case(f"input_{k}_bytes", 6, "raw", bytes(k)))
    out.append(raw("windowisempty_first_rep", 6, [rep(0, 2)], known=False))
    return out


def lzma2_cases():
    S, C = W.Stored, W.Chunk
    t = text(3000, 6000)
    out = []
    first = C(lits(t[:200]) + [match(20, 30)], reset=3, props=(3, 0, 2))
    # control classes and first-chunk forms
    out.append(lzma2("l2_empty", 7, [], liblzma=True))
    out.append(lzma2("l2_reset3_first", 7, [first], liblzma=True))
    out.append(lzma2("l2_reset0_first_traps", 7, [C(lits(t[:50]), reset=0)]))
    out.append(lzma2("l2_reset1_first_defaults", 7, [C(lits(t[:50]) + [match(5, 9)], reset=1)]))
    out.append(lzma2("l2_reset2_first", 7, [C(lits(t[:50]), reset=2, props=(0, 4, 0))]))
    out.append(lzma2("l2_stored1_first", 7, [S(t[:100], True), C(lits(t[100:150]) + [match(30, 120)], reset=2, props=(3, 0, 2))], liblzma=True))
    out.append(lzma2("l2_stored2_first", 7, [S(t[:100], False), C(lits(t[100:150]), reset=2, props=(3, 0, 2))]))
    for cb in (3, 0x10, 0x7F):
        out.append(lzma2(f"l2_control_{cb}", 7, [first, S(b"q", control=cb)]))
    for r in range(4):
        out.append(lzma2(f"l2_second_chunk_reset{r}", 7, [first, C(lits(t[200:260]) + [match(40, 150), rep(0, 5)], reset=r,
                                                                    props=(1, 3, 1))], liblzma=r in (1, 2)))
    out.append(lzma2("l2_reset2_new_props_same_dict", 7, [first, C([match(100, 180), lit(3)], reset=2, props=(0, 0, 4))]))
    out.append(lzma2("l2_state_reps_across_stored", 7, [C(lits(t[:100]) + [match(10, 40), rep(1, 3)], reset=3), S(t[:64], False),
                                                        C([rep(0, 4), lit_vs_match(2), rep(1, 5)], reset=0)]))
    # dictionary resets
    for how, pre in (("stored", [first, S(b"X" * 10, True)]), ("chunk", [first])):
        nxt = 3 if how == "chunk" else 0
        out.append(lzma2(f"l2_dict_reset_{how}_literal", 7, pre + [C(lits(b"\xFFAB"), reset=nxt)]))
        out.append(lzma2(f"l2_dict_reset_{how}_rep", 7, pre + [C([rep(0, 2)], reset=nxt)]))
        out.append(lzma2(f"l2_dict_reset_{how}_short_rep", 7, pre + [C([SHORT], reset=nxt)]))
        out.append(lzma2(f"l2_dict_reset_{how}_match_behind", 7, pre + [C([match(8, 150)], reset=nxt)]))
    # wrong sizes
    out.append(lzma2("l2_unpack_too_large", 7, [C(lits(t[:80]) + [end()], reset=3, unpack=81)]))
    m = W.Model()
    m.reset()
    clen = len(W.encode_ops(m, lits(t[:80])))
    out.append(lzma2("l2_comp_plus_1", 7, [C(lits(t[:80]), reset=3, comp=clen + 1)]))
    out.append(lzma2("l2_comp_minus_1", 7, [C(lits(t[:80]), reset=3, comp=clen - 1)]))
    out.append(lzma2("l2_unpack_minus_1", 7, [C(lits(t[:80]), reset=3, unpack=79)]))
    out.append(lzma2("l2_props_225", 7, [C(lits(t[:8]), reset=2, props=225)]))
    out.append(lzma2("l2_props_lc8_lp4", 7, [C(lits(b"\xFF" * 32 + t[:200]) + [match(20, 7)], reset=3, props=(8, 4, 4))]))
    out.append(lzma2("l2_props_lc4_lp1_after_small", 7, [first, C(lits(t[300:400]), reset=2, props=(4, 1, 2)),
                                                         C(lits(t[400:420]) + [rep(0, 6)], reset=0)]))
    # stored chunk sizes
    for n in (1, 2, 127, 128, 129, 65535, 65536):
        out.append(lzma2(f"l2_stored_{n}", 7, [S((t * 30)[:n], True), C([match(3, n - 1 if n > 1 else 0)], reset=3)]))
    # big chunks: 2 MiB unpacked, ~64 KiB packed
    out.append(lzma2("l2_chunk_2_mib_unpacked", 7, [C(lits(t[:100]) + [match(273, 99)] + [rep(0, 273)] * ((2 * MIB - 373) // 273)
                                                      + lits(b"e" * ((2 * MIB - 373) % 273)), reset=3)], dict_byte=24, liblzma=True))
    rnd = random.Random(6001)
    out.append(lzma2("l2_chunk_64k_packed", 7, [C(lits(bytes(rnd.randrange(256) for _ in range(64000))), reset=3)], dict_byte=24,
                     liblzma=True))
    # dictionary bytes
    for db in list(range(64)) + [0x40, 0x80, 0xC0, 0xFF]:
        ds = W.lzma2_dict_size(db)
        if db == 0:
            out.append(lzma2("l2_dict_0_match_4095", 7, [S((t * 2)[:5000], True), C([match(3, 4095)], reset=3)], dict_byte=0))
            out.append(lzma2("l2_dict_0_match_4096", 7, [S((t * 2)[:5000], True), C([match(3, 4096)], reset=3)], dict_byte=0))
        out.append(lzma2(f"l2_dict_byte_{db}", 7, [S(t[:50], True), C([match(10, 20)], reset=2, props=(3, 0, 2))], dict_byte=db,
                         liblzma=ds is not None and db <= 30))
    return out


def residues():
    """chunk boundaries and stream ends at stream offsets 0, 1, 126 and 127 modulo 128 (the kernel reads 128-byte windows;
    the single-stream API starts the chunks one byte in, behind the dictionary byte)"""
    out = []
    t = text(2000, 7000)
    for r in (0, 1, 126, 127):
        chunks = []
        pos = 0
        for j in range(3):
            want = (j + 1) * 256 + r          # next control byte offset
            n = want - pos - 3
            chunks.append(W.Stored(t[pos % 500:pos % 500 + n], j == 0))
            pos = want
        chunks.append(W.Chunk(lits(t[:30]) + [match(50, 400)], reset=2, props=(3, 0, 2)))
        out.append(lzma2(f"l2_boundaries_at_{r}", 8, chunks, liblzma=True))
        # a whole stream ending at residue r: stored padding in front of an LZMA chunk
        m = W.Model(dict_size=1 << 20)
        m.reset()
        body = len(W.encode_ops(m, lits(t[:40]) + [match(20, 30)]))
        pad = (r - (3 + 6 + body + 1)) % 128 + 128
        out.append(lzma2(f"l2_stream_ends_at_{r}", 8, [W.Stored(t[:pad], True), W.Chunk(lits(t[:40]) + [match(20, 30)], reset=3)]))
    return out


_CAT = None


def catalogue():
    global _CAT
    if _CAT is None:
        _CAT = properties() + dictionaries() + pos_slots() + lengths() + states() + termination() + lzma2_cases() + residues()
        names = [c.name for c in _CAT]
        assert len(set(names)) == len(names)
    return _CAT


class Cut:
    __slots__ = ("name", "case", "data", "tail")

    def __init__(self, name, case, data, tail):
        self.name, self.case, self.data, self.tail = name, case, data, tail


def truncations(limit=160):
    """every proper prefix of each case of at most `limit` bytes that decodes"""
    out = []
    for c in catalogue():
        if c.status != W.OK or len(c.data) > limit:
            continue
        for k in range(len(c.data)):
            out.append(Cut(f"{c.name}[:{k}]", c, c.data[:k], c.data[k:]))
    return out
