"""The hand-built Deflate catalogue (tests/deflate_cases.py) on the CPU: the oracle decodes every case to its intended
bytes and consumes exactly the stream (or fails with the status the case names), zlib agrees on every case RFC 1951
allows, every truncation fails, and the traces still cover the decoder limits the catalogue exists for."""
import os
import re
import zlib

import pytest

import deflate_cases as D
from deflate_writer import (DIST_BASE, LEN_BASE, LEN_EXTRA, DIST_EXTRA, K1W_WIN_BITS, K1W_WIN_WORDS, Code, DeflateWriter,
                            Match, k1w_window_offsets, oversubscribe, staircase)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cases():
    return D.catalogue()


def _valid(cases, plain=False):
    return [c for c in cases if c.expect is not None and not (plain and c.family == 7)]


def test_oracle_decodes_every_case(oracle, cases):
    bad = []
    for c in cases:
        st, out, used = oracle.deflate_decompress(c.data, c.start_bit)
        if c.expect is None:
            if st != c.status:
                bad.append((c.name, st, c.status))
        elif (st, out, used) != (0, c.expect, c.nbits):
            bad.append((c.name, st, len(out), len(c.expect), used, c.nbits))
    assert not bad, f"{len(bad)} of {len(cases)} cases differ from the oracle: {bad[:8]}"


def test_zlib_agrees_where_rfc1951_allows(cases):
    """zlib owes nothing to the reference: it ties the writer and the oracle to RFC 1951.  Where the case names a rule
    under which zlib rejects the stream, zlib must reject it."""
    bad = []
    for c in _valid(cases):
        assert not (c.stored and c.start_bit)
        v = int.from_bytes(c.data[:c.stream_bytes], "little") >> c.start_bit
        stream = v.to_bytes((c.nbits + 7) // 8, "little") + c.data[c.stream_bytes:]
        trailing = c.data[c.stream_bytes:]
        d = zlib.decompressobj(-15)
        try:
            out = d.decompress(stream) + d.flush()
            ok = d.eof and out == c.expect and d.unused_data == trailing
        except zlib.error:
            ok = False
        if ok != (c.zlib is True):
            bad.append((c.name, c.zlib))
    assert not bad, f"zlib disagrees with {len(bad)} cases: {bad[:8]}"


def test_every_truncation_fails(oracle):
    """Every compact case cut at every byte (and shifted by 0..7 start bits) fails: symbolNotFound, the trap for fewer
    than 3 header bits, a stored-length error, or wrongBlockType for fewer than 10 bits."""
    units = D.truncation_units()
    assert len(units) > 20000
    seen = set()
    for t in units:
        st, _, _ = oracle.deflate_decompress(t.data, t.start_bit)
        assert st in (D.NOT_FOUND, D.TRAP, D.BAD_STORED, D.BAD_BTYPE), (t.name, st)
        seen.add(st)
    assert seen == {D.NOT_FOUND, D.TRAP, D.BAD_STORED, D.BAD_BTYPE}


# ----------------------------------------------------------------------------------------------- writer
def test_code_assignment_matches_rfc1951_for_complete_sets():
    """RFC 1951 3.2.2 example: lengths (3, 3, 3, 3, 3, 2, 4, 4) -> codes 010 011 100 101 110 00 1110 1111"""
    c = Code([3, 3, 3, 3, 3, 2, 4, 4])
    assert [c.codes[s] for s in range(8)] == [0b010, 0b011, 0b100, 0b101, 0b110, 0b00, 0b1110, 0b1111]
    assert all(c.reads_back(s) for s in range(8))


def test_oversubscribed_code_wraps_behind_a_shorter_prefix():
    lens = staircase([5, 1, 9, 3])                      # 5:1 1:2 9:3 3:3
    over = oversubscribe(lens, 12)
    c = Code([over.get(s, 0) for s in range(12)])
    assert c.kraft > 1 and all(c.reads_back(s) for s in lens) and not c.reads_back(11)
    with pytest.raises(ValueError):
        w = DeflateWriter()
        w.dynamic([11], [over.get(s, 0) for s in range(12)] + [0] * 244 + [1], [1, 1])


def test_writer_records_matches_and_runs():
    w = DeflateWriter(start_bits=3, junk=5)
    w.fixed([b"abcd" * 70, Match(258, 4, 284, 31), 120, Match(3, 1)], final=True)
    (l1, d1, r1, s1, x1, _, _, p1, e1), (_, _, r2, s2, _, _, _, _, _) = w.trace.matches
    assert (l1, d1, r1, s1, x1, r2, s2) == (258, 4, 280, 284, 31, 1, 257)
    assert p1 == 3 + 3 + 280 * 8 and e1 - p1 == 8 + 5 + 5          # 284 + 5 extra bits, distance code 3 (no extra bits)
    assert w.out == b"abcd" * 70 + b"abcd" * 64 + b"ab" + b"xxxx"


# ----------------------------------------------------------------------------------------------- coverage contract
def _lengths(cases, family=None):
    out = set()
    for c in _valid(cases, plain=True):
        if family is None or c.family == family:
            out |= c.trace.lengths
    return out


def test_coverage_every_code_length_and_all_ones_code(cases):
    lens = _lengths(cases)
    for a in ("lit", "dist"):
        assert {L for b, L in lens if b == a} >= set(range(1, 16)), a
    assert {"lit", "dist"} <= set().union(*(c.trace.all_ones for c in _valid(cases, plain=True)))
    # the all-ones code as a literal, a length symbol and end of block
    ones = {(s[0], s[1]) for c in _valid(cases, plain=True) for s in c.trace.symbols if s[2] == 15}
    lit_ones = {s for a, s in ones if a == "lit"}
    assert {121, 284, 256} <= lit_ones


def test_coverage_lut_boundaries(cases):
    """both sides of K1L's 7|8 (lit/len) and 5|6 (distance) lookup limits and K1w's 11|12 and 9|10"""
    lens = _lengths(cases)
    for a, cut in (("lit", 7), ("lit", 11), ("dist", 5), ("dist", 9)):
        assert (a, cut) in lens and (a, cut + 1) in lens


def test_coverage_every_length_and_distance_symbol(cases):
    ls, ds, dists = set(), set(), set()
    for c in _valid(cases, plain=True):
        for m in c.trace.matches:
            ls.add((m[3], m[4]))
            ds.add((m[5], m[6]))
            dists.add(m[1])
    for s in range(257, 285):
        assert (s, 0) in ls and (s, (1 << D.LEN_EXTRA[s - 257]) - 1) in ls, s
    assert (285, 0) in ls and (284, 31) in ls                       # 258 both ways
    for d in range(30):
        assert (d, 0) in ds and (d, (1 << D.DIST_EXTRA[d]) - 1) in ds, d
    assert 32768 in dists


def test_coverage_literal_runs(cases):
    runs = {m[2] for c in _valid(cases, plain=True) for m in c.trace.matches}
    assert set(D.RUNS) <= runs
    # each threshold also through stored, fixed and dynamic blocks and a run that crosses all three
    for n in D.RUNS:
        for how in ("stored", "fixed", "dynamic", "mixed"):
            c = next(c for c in cases if c.name == f"run_{n}_{how}")
            assert c.trace.matches[0][2] == n


def test_coverage_overlapping_matches_at_every_word_residue(cases):
    seen = set()
    for c in _valid(cases, plain=True):
        if not c.name.startswith("overlap_"):
            continue
        pos = 0                                      # output position of each match, from the runs before them
        for m in c.trace.matches:
            pos += m[2]
            seen.add((m[1], m[0], pos % 8))
            pos += m[0]
    for d in range(1, 9):
        for ln in list(range(3, 11)) + [258]:
            assert {(d, ln, r) for r in range(8)} <= seen, (d, ln)


def test_coverage_k1w_windows(cases):
    """48-bit symbols (15-bit length code + 5 extra bits + 15-bit distance code + 13 extra bits) start at every one of
    the 608 bit offsets of a warp-decoder window, and on both sides of a chunk end"""
    offs, crossing, later = set(), 0, 0
    for c in _valid(cases, plain=True):
        if not c.name.startswith("w48_"):
            continue
        for b in c.trace.blocks:
            if b[0] != "dynamic":
                continue
            for m, (off, chunk, crosses) in zip([m for m in c.trace.matches if b[2] <= m[7] < b[3]],
                                                k1w_window_offsets(c.trace, b)):
                if m[8] - m[7] == 48:
                    offs.add(off)
                    crossing += crosses
                    later += chunk > 0
    assert offs == set(range(608))
    assert crossing >= 3 and later > 0


def test_coverage_nosync_stream(cases):
    c = next(c for c in cases if c.name == "nosync_8bit")
    assert c.nbits > 2 * 32 * 608                         # several chunks of windows that never fall into step


def test_coverage_oversubscribed_sets_still_decode(cases):
    """the slow kernel's success path: over-subscribed lit/len, distance and code-length sets that decode to the intended
    bytes"""
    over = set()
    for c in _valid(cases):
        if c.family == 7:
            for b in c.trace.blocks:
                over |= set(b[4])
    assert over == {"lit", "dist", "cl"}
    names = {c.name.split("/")[0] for c in cases if c.family == 7}
    plain = {c.name for c in _valid(cases, plain=True) if c.family in (1, 3, 4) and c.name != "hazard_dist_30_31"}
    assert names == plain


def test_coverage_truncations_end_inside_long_fields():
    """Some truncation ends strictly inside a 15-bit code of each alphabet, inside length extra bits 5 wide, distance
    extra bits 7 and 13 wide, and a 48-bit match: the decoders' lazy end-of-input checks meet every long field."""
    fields = {}
    for t in D.truncation_units():
        c = t.case
        if c.name not in fields:
            k = c.start_bit
            f = [(f"{a}15", p - k, p - k + 15) for a, _, L, p in c.trace.symbols if L == 15 and a in ("lit", "dist")]
            f += [(f"{a}x{w}", p - k, p - k + w) for a, w, p in c.trace.extras if (a, w) in (("lit", 5), ("dist", 7), ("dist", 13))]
            f += [("m48", m[7] - k, m[8] - k) for m in c.trace.matches if m[8] - m[7] == 48]
            fields[c.name] = (f, set())
        fields[c.name][1].add(t.avail)
    hit = set()
    for f, avail in fields.values():
        for kind, a, b in f:
            if any(a < x < b for x in avail):
                hit.add(kind)
    assert hit == {"lit15", "dist15", "litx5", "distx7", "distx13", "m48"}, hit


# ----------------------------------------------------------------------------------------------- misaligned parses
class _Parser:
    """Reads a block's symbols with its codes from any bit offset, the way the oracle's decoder would (shortest prefix,
    the code assigned last on a path)."""

    def __init__(self, case, block):
        self.bits = "".join(format(b, "08b")[::-1] for b in case.data)
        self.lit, self.dist = [{(L, c): s for (L, c), s in code.slots.items()} for code in case.trace.codes[block[2]]]
        self.end = block[3]

    def _sym(self, tab, p):
        c = 0
        for L in range(1, 16):
            if p + L > len(self.bits):
                return None, p
            c = (c << 1) | (self.bits[p + L - 1] == "1")
            if (L, c) in tab:
                return tab[(L, c)], p + L
        return None, p

    def _int(self, p, n):
        return int(self.bits[p:p + n][::-1] or "0", 2), p + n

    def token(self, p):
        """-> (kind, output bytes, distance, next bit): kind 'lit', 'match', 'eob', 'not_found', 'wrong_lit', 'wrong_dist'"""
        s, p = self._sym(self.lit, p)
        if s is None:
            return "not_found", 0, 0, p
        if s < 256:
            return "lit", 1, 0, p
        if s == 256:
            return "eob", 0, 0, p
        if s > 285:
            return "wrong_lit", 0, 0, p
        x, p = self._int(p, LEN_EXTRA[s - 257])
        d, p = self._sym(self.dist, p)
        if d is None:
            return "not_found", 0, 0, p
        if d > 29:
            return "wrong_dist", 0, 0, p
        y, p = self._int(p, DIST_EXTRA[d])
        return "match", LEN_BASE[s - 257] + x, DIST_BASE[d] + y, p

    def true_chain(self, p0):
        """-> {token start: output bytes before it}"""
        starts, out, p = {}, 0, p0
        while True:
            starts[p] = out
            kind, n, _, p = self.token(p)
            assert kind in ("lit", "match", "eob")
            out += n
            if kind == "eob":
                return starts


def _misparse_stops(case, span=4096):
    """what stops a parse that starts at each bit offset of the block's first `span` bits that is not a token start,
    before it falls into step with the true chain"""
    block = next(b for b in case.trace.blocks if b[2] is not None and b[3] - b[2] > span)
    P = _Parser(case, block)
    starts = P.true_chain(block[2])
    before = sorted(starts.items())
    kinds = set()
    for s in range(block[2], block[2] + span):
        if s in starts:
            continue
        out = max(o for q, o in before if q < s)                # output of the true tokens before the guessed start
        p = s
        for _ in range(400):
            if p in starts:
                kind = "sync"
                break
            kind, n, d, p = P.token(p)
            if kind == "match" and d > out:
                kind = "past_output"
            if kind not in ("lit", "match"):
                break
            out += n
        kinds.add(kind)
    return kinds


@pytest.mark.parametrize("name,stops", [("hazard_fixed_286_287", {"wrong_lit", "wrong_dist", "eob"}),
                                        ("hazard_short_eob", {"eob"}),
                                        ("hazard_near_start", {"past_output"}),
                                        ("hazard_dist_30_31", {"wrong_dist"})])
def test_hazard_misparses_meet_what_they_claim(cases, name, stops):
    c = next(c for c in cases if c.name == name)
    kinds = _misparse_stops(c)
    assert stops <= kinds and "sync" in kinds, kinds


def test_k1w_model_matches_the_kernel():
    """the window model of the coverage contract uses inflate_warp.cu's window size"""
    with open(os.path.join(ROOT, "swcompression_b200", "csrc", "inflate_warp.cu")) as f:
        src = f.read()
    assert int(re.search(r"constexpr int WIN_WORDS = (\d+);", src).group(1)) == K1W_WIN_WORDS
    assert re.search(r"for \(int round = 0; round < 33; round\+\+\)", src)


def test_nosync_stream_drives_pass_a_to_its_round_limit(cases):
    """The warp decoder's pass A on the first chunk of nosync_8bit: lane i starts at i windows, a lane restarts where its
    predecessor ended, until nothing changes.  Wrongly started lanes never fall into step, so the true start has to walk
    lane by lane: about 32 rounds of the 33 allowed."""
    c = next(c for c in cases if c.name == "nosync_8bit")
    block = next(b for b in c.trace.blocks if b[0] == "dynamic")
    P = _Parser(c, block)
    base, W = block[2], K1W_WIN_BITS

    def window(start, hi):
        p = start
        while True:
            kind, _, _, p = P.token(p)
            if kind not in ("lit", "match"):
                return p, True
            if p >= hi:
                return p, False

    start = [base + i * W for i in range(32)]
    valid, dirty, res = [True] * 32, [True] * 32, [None] * 32
    for rnd in range(33):
        for i in range(32):
            if dirty[i] and valid[i]:
                res[i] = window(start[i], base + (i + 1) * W)
        nvalid = [True] + [valid[i - 1] and not res[i - 1][1] for i in range(1, 32)]
        nstart = [start[0]] + [res[i - 1][0] for i in range(1, 32)]
        dirty = [nvalid[i] != valid[i] or (nvalid[i] and nstart[i] != start[i]) for i in range(32)]
        valid, start = nvalid, nstart
        if not any(dirty):
            break
    assert rnd + 1 >= 30, f"pass A settled after {rnd + 1} rounds"
