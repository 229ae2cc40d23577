"""A named catalogue of hand-built LZ4 blocks and frames (written by tests/lz4_writer.py) and every byte cut of its small
blocks.  Each case carries the reference's answer from the writer's model of the Swift decoder.  Families 1-7 are raw
blocks (with the case's dictionary, or none); family 8 is whole frames with dependent blocks."""
import random

import lz4_writer as W
from lz4_writer import FBlock, Seq

MIB = 1 << 20
F24 = 1 << 24
DICT_LENGTHS = (0, 1, 3, 4096, 65535, 65536, 100000)
_DICTS = {}


def rb(n, seed):
    """n deterministic pseudo-random bytes"""
    return random.Random(seed).randbytes(n)


def dictionary(length):
    """the family 7 dictionary of `length` bytes (0: empty but present)"""
    if length not in _DICTS:
        _DICTS[length] = rb(length, 7000 + length)
    return _DICTS[length]


class Case:
    """form "block": `data` is a raw block decoded with `dictionary` (None: no dictionary); form "frame": `data` is a whole
    LZ4 stream for LZ4.decompress / LZ4.multiDecompress with `dictionary`."""

    def __init__(self, name, family, data, dictionary=None, form="block"):
        self.name, self.family, self.data, self.dictionary, self.form = name, family, bytes(data), dictionary, form
        if form == "block":
            self.model = W.decode_block(self.data, dictionary)
            self.status = self.model.status
            self.out = self.model.out
        else:
            self.model = W.decode(self.data, dictionary)
            self.status = self.model.status
            self.out = self.model.out
            self.multi = W.multi_decode(self.data, dictionary)
        # the runs as the one-kernel decoder's window sees them when the block is the first of a dependent frame (whose
        # dictionary is cut to its last 64 KiB)
        small = form == "block" and len(self.data) <= 4 * MIB
        self.lanes = W.kernel_window_runs(self.data, min(len(dictionary or b""), W.WINDOW)) if small else []

    @property
    def dict_key(self):
        return None if self.dictionary is None else len(self.dictionary)


def prefix_seqs(p, seed):
    """sequences of 4..17 bytes each (1..14 literals, a 4-byte match at offset 1) that fill exactly `p` bytes (p = 0 or
    p >= 4)"""
    out, k = [], 0
    while p > 0:
        s = p if p <= 17 else min(17, p - 4)
        out.append(Seq(rb(s - 3, seed * 100 + k), 4, 1))
        p -= s
        k += 1
    return out


def placed(r, inner, body, seed):
    """`body` sequences behind a prefix that puts byte `inner` of the body at block position = r (mod 32)"""
    p = (r - inner) % 32
    if 0 < p < 4:
        p += 32
    return prefix_seqs(p, seed) + body


def run_lengths(r):
    """extension runs tried at block position r (mod 32): one byte, the runs whose last byte or terminator sits at the
    next multiple of 32, runs across one and two such boundaries, and 70 bytes"""
    return sorted({1, 32 - r, 33 - r, 64 - r, 65 - r, 70} - {0})


def run_grid(step):
    """(residue, run length) pairs: run_lengths(r) at every residue, and every length 1..70 at a residue that moves by
    `step`"""
    pairs = {(r, k) for r in range(32) for k in run_lengths(r)} | {((k * step) % 32, k) for k in range(1, 71)}
    return sorted(pairs)


def run_value(k, t):
    """the field value (past the nibble's 15) of a run of k bytes ending in terminator t"""
    return 255 * (k - 1) + t


# -------------------------------------------------------------------------------------------------------- family 1
def literal_field():
    cases = []
    tail = Seq(rb(12, 1))
    for n in list(range(17)) + [269, 270, 271, 524, 525]:
        lit = rb(n, 100 + n)
        cases.append(Case(f"lit_{n}_final", 1, W.write_block([Seq(rb(20, 2), 4, 1), Seq(lit + rb(max(0, 5 - n), 3))])))
        if n:
            cases.append(Case(f"lit_{n}_mid", 1, W.write_block([Seq(lit, 4 + n % 7, 1 + n % max(n, 1)), tail])))
        cases.append(Case(f"lit_{n}_single", 1, W.write_block([Seq(lit)])))
    for r, k in run_grid(11):
        v = 15 + run_value(k, (r * 37 + k) % 255)
        body = [Seq(rb(v, 200 + r * 100 + k), 5, 3), tail]
        cases.append(Case(f"lit_run_{k}_at_{r}", 1, W.write_block(placed(r, 1, body, r))))
        if k <= 2:
            body = [Seq(rb(v, 300 + r * 100 + k))]
            cases.append(Case(f"lit_run_{k}_at_{r}_final", 1, W.write_block(placed(r, 1, body, r))))
    # runs that end in 255 where the block ends, and a 255 run followed by its terminator as the last byte
    for k in (1, 2, 31, 32, 33):
        pre = W.write_block([Seq(rb(6, 4), 4, 1)])
        cases.append(Case(f"lit_run_{k}_off_block", 1, pre + bytes([0xF0]) + b"\xFF" * k))
        cases.append(Case(f"lit_run_{k}_terminated_last_byte", 1, pre + bytes([0xF0]) + b"\xFF" * k + b"\x00"))
    return cases


# -------------------------------------------------------------------------------------------------------- family 2
def match_field():
    cases = []
    tail = Seq(rb(12, 5))
    for m in list(range(4, 20)) + [273, 274, 528, 529]:
        cases.append(Case(f"mlen_{m}", 2, W.write_block([Seq(rb(8, 6), m, 1 + m % 8), tail])))
    for r, k in run_grid(13):
        m = 19 + run_value(k, (r * 41 + k) % 255)
        body = [Seq(rb(8, 400 + r), m, 1 + (r + k) % 8), tail]
        cases.append(Case(f"mlen_run_{k}_at_{r}", 2, W.write_block(placed(r, 11, body, 50 + r))))
    for k in (1, 2, 31, 32, 33):
        pre = W.write_block([Seq(rb(6, 7), 4, 1)])
        cases.append(Case(f"mlen_run_{k}_off_block", 2, pre + bytes([0x1F]) + b"x\x01\x00" + b"\xFF" * k))
    return cases


def window_lanes(field):
    """a run of `field` at every lane of the one-kernel decoder's window (W.kernel_window_runs) that it can reach, as a
    one-byte run inside the window and a 40-byte run across it.  The lane is set by where the window was last re-based
    (at a token, an offset or a run), so the runs sit behind a first sequence of 1..70 literals and a 4, 19 or 300-byte
    match, and a match run behind 0..28 literals of its own sequence.  A match run never starts at lane 1: the offset's
    two bytes are in the window in front of it, or it opens a new window at lane 0."""
    cases, todo = [], set(range(32)) - ({1} if field == "mlen" else set())
    tail = Seq(rb(12, 60))
    for q in range(1, 71):
        for pm in (4, 19, 300):
            for a in (range(29) if field == "mlen" else [None]):
                def build(k):
                    if field == "lit":
                        test = Seq(rb(15 + run_value(k, 99), 61), 4, 1)
                    else:
                        test = Seq(rb(a, 62), 19 + run_value(k, 99), 1)
                    return W.write_block([Seq(rb(q, 63), pm, 1), test, tail])
                lane = W.kernel_window_runs(build(1))[-1][1]
                if lane not in todo:
                    continue
                todo.discard(lane)
                for k in (1, 40):
                    blk = build(k)
                    assert W.kernel_window_runs(blk)[-1][:3] == (field, lane, k)
                    cases.append(Case(f"{field}_run_{k}_lane_{lane}", 1 if field == "lit" else 2, blk))
    assert not todo, (field, todo)
    return cases


# -------------------------------------------------------------------------------------------------------- family 3
OFFSETS = list(range(1, 18)) + [31, 32, 33, 63, 64, 65, 511, 512, 513, 65535]
MLENS = [4, 5, 31, 32, 33, 63, 64, 65, 300, 70000]


def offsets():
    cases = []
    tail = Seq(rb(12, 8))
    grid = {(o, m) for o in OFFSETS for m in (4, 5, 33, 65, 300)} | {(o, m) for o in (1, 2, 3, 7, 16, 17, 32, 512) for m in MLENS}
    for o, m in sorted(grid):
        lit = rb(max(o, 20), 500 + o)
        cases.append(Case(f"offset_{o}_mlen_{m}", 3, W.write_block([Seq(lit, m, o), tail])))
    for op in (1, 5, 100, 65535):
        lit = rb(op, 600 + op)
        for d, what in ((0, "eq"), (1, "plus1")):
            if op + d <= 65535:
                cases.append(Case(f"offset_{what}_op_{op}", 3, W.write_block([Seq(lit, 8, op + d), tail])))
        cases.append(Case(f"offset_0_op_{op}", 3, W.write_block([Seq(lit, 8, 0), tail])))
    # a match whose offset equals the whole output so far, later in the block
    cases.append(Case("offset_eq_op_third_seq", 3, W.write_block([Seq(rb(9, 9), 6, 2), Seq(rb(3, 10), 4, 18), tail])))
    cases.append(Case("offset_plus1_third_seq", 3, W.write_block([Seq(rb(9, 9), 6, 2), Seq(rb(3, 10), 4, 19), tail])))
    return cases


# -------------------------------------------------------------------------------------------------------- family 4
def end_of_block():
    cases = [Case("empty_block", 4, b"")]
    for n in range(5):
        cases.append(Case(f"single_{n}_literals", 4, W.write_block([Seq(rb(n, 11))])))
    for n in range(6):
        cases.append(Case(f"final_{n}_after_match", 4, W.write_block([Seq(rb(20, 12), 12, 1), Seq(rb(n, 13))])))
    for m, n in ((6, 5), (7, 5), (8, 4), (7, 4), (6, 6), (7, 6), (19, 4), (4, 8), (4, 7), (300, 5)):
        # the last match starts m + n bytes before the end: 11 against 12, alone and with the literal rule
        cases.append(Case(f"last_match_{m + n}_before_end_final_{n}", 4, W.write_block([Seq(rb(20, 14), m, 1), Seq(rb(n, 15))])))
    cases.append(Case("last_match_11_then_empty_seq", 4, W.write_block([Seq(rb(20, 16), 6, 1), Seq(b"", 4, 1), Seq(rb(12, 17))])))
    cases.append(Case("earlier_match_near_end_later_far", 4,
                      W.write_block([Seq(rb(20, 16), 6, 1), Seq(rb(3, 18), 9, 2), Seq(rb(5, 19))])))
    cases.append(Case("ends_after_match", 4, W.write_block([Seq(rb(20, 20), 12, 1)])))
    # cuts at named places of one block: after the token, inside the offset, inside each extension run, inside literals
    full = W.write_block([Seq(rb(40, 21), 300, 7), Seq(rb(12, 22))])
    named = {"after_token": 1, "inside_literals": 2 + 20, "before_offset": 2 + 40,
             "inside_offset": 2 + 40 + 1, "before_mlen_ext": 2 + 40 + 2, "inside_mlen_ext": 2 + 40 + 3,
             "after_match": 2 + 40 + 2 + 2, "after_final_token": 2 + 40 + 2 + 2 + 1}
    assert full[1] == 25 and full[44] == 255 and full[45] == 26
    for what, k in named.items():
        cases.append(Case(f"cut_{what}", 4, full[:k]))
    # the lit extension byte alone (token 0xF7, its run cut before the terminator)
    cases.append(Case("cut_inside_lit_run", 4, bytes([0xF7]) + b"\xFF\xFF"))
    return cases


# -------------------------------------------------------------------------------------------------------- family 5
def record_fields():
    """lit and mlen at 2^24 - 1 (the largest the parse kernel's 24-bit records hold) and 2^24 (the fallback kernel's)"""
    cases = []
    tail = Seq(rb(12, 23))
    for v in (F24 - 1, F24):
        lit = rb(v, 24)
        cases.append(Case(f"lit_{v}_mid", 5, W.write_block([Seq(lit, 4, 1), tail])))
        cases.append(Case(f"lit_{v}_final", 5, W.write_block([Seq(rb(20, 25), 4, 1), Seq(lit)])))
        cases.append(Case(f"mlen_{v}_mid", 5, W.write_block([Seq(rb(8, 26), v, 3), tail])))
        cases.append(Case(f"mlen_{v}_then_short", 5, W.write_block([Seq(rb(8, 27), v, 1), Seq(rb(3, 28), 9, 5), tail])))
    big = rb(F24, 29)
    cases.append(Case("lit_and_mlen_mixed", 5, W.write_block([Seq(big, F24 - 1, 65535), Seq(big[:F24 - 1], F24, 700),
                                                              Seq(rb(5, 30), 40, 9), Seq(big[:F24 - 1])])))
    return cases


# -------------------------------------------------------------------------------------------------------- family 6
def scheduling():
    cases = []
    tail = Seq(rb(12, 31))
    for nrec in (31, 32, 33, 63, 64, 65):
        seqs = [Seq(rb(1 + j % 5, 3100 + j), 4 + j % 9, 1 + j % 6) for j in range(nrec - 1)]
        cases.append(Case(f"records_{nrec}", 6, W.write_block(seqs + [tail])))
    # every match reads the one before it (1 literal between: offset 1 + its length)
    for m, label in ((8, "copy"), (20, "overlap")):
        seqs = [Seq(rb(16, 32), 8, 1)]
        for j in range(1, 70):
            seqs.append(Seq(rb(1, 3200 + j), m, 9 if label == "copy" else 3))
        cases.append(Case(f"chain_all_{label}", 6, W.write_block(seqs + [tail])))
    # one dependent match at record t, the others reading the first literal run
    for t in list(range(1, 40)) + [63, 64, 65]:
        seqs, op = [Seq(rb(64, 33), 6, 5)], 70
        prev_end = 70
        for j in range(1, t + 2):
            lit = rb(2, 3300 + j)
            op += 2
            if j == t:
                mlen, off = 8, op - (prev_end - 8)          # the previous match's output
            else:
                mlen, off = 4 + j % 20, op - (j % 40)
            seqs.append(Seq(lit, mlen, off))
            op += mlen
            prev_end = op
        cases.append(Case(f"dependent_at_{t}", 6, W.write_block(seqs + [tail])))
    # a long match (whole warp) read by the short ones behind it
    for t in (1, 6, 7, 8, 31, 32):
        seqs = [Seq(rb(30, 34), 4, 1) for _ in range(t - 1)] + [Seq(rb(30, 35), 100, 30)]
        for j in range(9):
            seqs.append(Seq(rb(1, 3400 + j), 5 + j, 20 + 14 * j))
        cases.append(Case(f"long_match_at_{t}_read_by_short", 6, W.write_block(seqs + [tail])))
    # literal runs of 63 / 64 / 65 at the records around the 8- and 32-record edges
    for n in (63, 64, 65):
        seqs = [Seq(rb(n if j in (7, 8, 31, 32) else 2, 3500 + j), 4 + j % 3, 1 + j % 4) for j in range(40)]
        cases.append(Case(f"literals_{n}_at_group_edges", 6, W.write_block(seqs + [tail])))
    return cases


# -------------------------------------------------------------------------------------------------------- family 7
def dictionaries():
    cases = []
    tail = Seq(rb(12, 36))
    for dl in DICT_LENGTHS:
        d = dictionary(dl)
        name = f"dict_{dl}"
        for op in (0, 4):
            lit = rb(op, 37)
            for delta, what in ((0, "eq"), (1, "plus1")):
                if op + dl + delta > 65535:
                    continue
                cases.append(Case(f"{name}_offset_{what}_op_{op}", 7, W.write_block([Seq(lit, 6, op + dl + delta), tail]), d))
        if dl == 0:
            continue
        reach = min(dl, 65535 - 4)
        for m in (4, 5, 33, 300):
            if m <= reach:
                cases.append(Case(f"{name}_inside_mlen_{m}", 7, W.write_block([Seq(rb(4, 38), m, 4 + reach), tail]), d))
        for into in (1, 2, 3, 20):
            if into <= dl:
                cases.append(Case(f"{name}_straddle_{into}", 7, W.write_block([Seq(rb(4, 39), 40, 4 + into), tail]), d))
        for off in (1, 2, 3):
            if off <= dl:
                cases.append(Case(f"{name}_overlap_from_start_{off}", 7, W.write_block([Seq(b"", 70, off), tail]), d))
        cases.append(Case(f"{name}_overlap_after_literals", 7, W.write_block([Seq(rb(2, 40), 33, 3), tail]), d))
        cases.append(Case(f"{name}_far", 7, W.write_block([Seq(b"", 4, min(dl, 65535)), Seq(rb(70, 41), 300, 65535 if dl >= 65465 else 70), tail]), d))
    return cases


# -------------------------------------------------------------------------------------------------------- family 8
def _fcase(name, blocks, d=None, **kw):
    return Case(name, 8, W.frame(blocks, **kw), d, form="frame")


def _cblock(seqs, last):
    return FBlock(W.block(seqs, last))


def chains():
    cases = []
    d = dictionary(4096)
    big = rb(70000, 42)
    # exactly 65 535 back across blocks
    for what in ("from_stored_block", "across_two_blocks"):
        first = [FBlock(big, stored=True)] if what == "from_stored_block" else [_cblock([], big[:65000]), _cblock([], big[65000:])]
        cases.append(_fcase(f"chain_back_65535_{what}", first + [_cblock([(b"", 20, 65535)], rb(12, 43))]))
    cases.append(_fcase("chain_window_after_short_block", [_cblock([], rb(10, 44)), _cblock([(b"", 6, 10)], rb(12, 45))], d))
    cases.append(_fcase("chain_beyond_short_block", [_cblock([], rb(10, 44)), _cblock([(b"", 6, 11)], rb(12, 45))], d))
    cases.append(_fcase("chain_into_stored_block", [FBlock(rb(100, 46), stored=True), _cblock([(rb(3, 47), 30, 53)], rb(12, 48))]))
    cases.append(_fcase("chain_zero_stored_then_dict", [FBlock(b"", stored=True), _cblock([(b"", 30, 100)], rb(12, 49))], d))
    cases.append(_fcase("chain_stored_then_dict_reach", [FBlock(rb(5, 50), stored=True), _cblock([(b"", 30, 100)], rb(12, 49))], d))
    cases.append(_fcase("chain_dict_first_block", [_cblock([(b"", 30, 4096)], rb(12, 51)), _cblock([(b"", 8, 40)], rb(12, 52))], d))
    cases.append(_fcase("chain_dict_second_block_refused", [_cblock([], rb(12, 53)), _cblock([(b"", 8, 100)], rb(12, 52))], d))
    cases.append(_fcase("chain_empty_dict_present", [_cblock([(rb(3, 54), 8, 3)], rb(12, 55))], b""))
    # 64 KiB dictionary window of a dependent frame: the first block may reach 65 535 into a 100 000-byte dictionary
    cases.append(_fcase("chain_dict_100000_window", [_cblock([(b"", 8, 65535)], rb(12, 56))], dictionary(100000)))
    cases.append(_fcase("independent_dict_each_block", [_cblock([(b"", 8, 4000)], rb(12, 57)), _cblock([(b"", 8, 4000)], rb(12, 58))],
                        d, independent=True))
    # block k fails (its final literal run is cut: truncated), a bad checksum on block k - 1, k or k + 1
    for nb in (1, 2, 33):
        for k in sorted({0, nb // 2, nb - 1}):
            for bad in (None, k - 1, k, k + 1):
                if bad is not None and not 0 <= bad < nb:
                    continue
                blocks = []
                for j in range(nb):
                    blk = W.block([(rb(3, 5900 + j), 9, 3 + 24 * min(j, 20))], rb(12, 6000 + j))
                    if j == k:
                        blk = blk[:-3]
                    blocks.append(FBlock(blk, ck=(0x12345678 if j == bad else None)))
                tag = "none" if bad is None else f"{bad - k:+d}"
                cases.append(_fcase(f"chain_{nb}_fail_{k}_badck_{tag}", blocks, block_checksums=True))
    # descriptor fields: content size, content checksum, dictionary ID
    good = [_cblock([(rb(3, 61), 9, 3)], rb(12, 62)), FBlock(rb(7, 63), stored=True)]
    want = W.decode(W.frame(good)).out
    cases.append(_fcase("chain_content_size", good, content_size=len(want)))
    cases.append(_fcase("chain_content_size_wrong", good, content_size=len(want) + 1))
    cases.append(_fcase("chain_content_checksum", good, content_checksum=want))
    cases.append(_fcase("chain_content_checksum_wrong", good, content_checksum=want + b"x"))
    cases.append(_fcase("chain_dict_id", good, d, dict_id=7))
    cases.append(_fcase("chain_dict_id_without_dict", good, None, dict_id=7))
    # several frames for multiDecompress: a dependent frame, a skippable one, a legacy one and an independent one
    multi = (W.frame([_cblock([(b"", 8, 50)], rb(12, 64))]) + b"\x50\x2A\x4D\x18\x03\x00\x00\x00abc" +
             W.legacy_frame([W.block([(rb(6, 65), 8, 2)], rb(12, 66))]) +
             W.frame([_cblock([(b"", 8, 60)], rb(12, 67))], independent=True))
    cases.append(Case("multi_frames_with_dict", 8, multi, d, form="frame"))
    cases.append(Case("multi_frames_truncated_last", 8, multi[:-2], d, form="frame"))
    return cases


_CAT = None


def catalogue():
    global _CAT
    if _CAT is None:
        _CAT = literal_field() + window_lanes("lit") + match_field() + window_lanes("mlen") + offsets() + end_of_block() + record_fields() + scheduling() + dictionaries() + chains()
        names = [c.name for c in _CAT]
        assert len(set(names)) == len(names), [n for n in names if names.count(n) > 1][:5]
    return _CAT


class Cut:
    __slots__ = ("name", "case", "data", "tail", "model")

    def __init__(self, name, case, data, tail):
        self.name, self.case, self.data, self.tail = name, case, data, tail
        self.model = W.decode_block(data, case.dictionary)


def truncations(limit=400):
    """every proper prefix of each block case of at most `limit` bytes that decodes, with the rest of the block behind it"""
    out = []
    for c in catalogue():
        if c.form != "block" or c.status != W.OK or len(c.data) > limit:
            continue
        for k in range(len(c.data)):
            out.append(Cut(f"{c.name}[:{k}]", c, c.data[:k], c.data[k:]))
    return out


def wrapped(c):
    """a block case as whole streams for LZ4.decompress -> [(form, stream, dictionary)]: the single block of a dependent
    B7 frame and of an independent one, both with the case's dictionary, and without a dictionary a legacy frame too.
    Blocks over 4 MiB (the largest frame block) have none."""
    if c.form != "block" or len(c.data) > 4 * MIB:
        return []
    out = [("dependent", W.frame([FBlock(c.data)], bd=0x70), c.dictionary),
           ("independent", W.frame([FBlock(c.data)], independent=True, bd=0x70), c.dictionary)]
    if c.dictionary is None:
        out.append(("legacy", W.legacy_frame([c.data]), None))
    return out


def past_4gib_block(count=257, mlen=F24 - 1):
    """`count` sequences of one literal and an offset-1 match of `mlen` bytes, then 12 literals -> (block, the value of each
    run of 1 + mlen equal bytes, the final literals).  At the defaults: 16.9 MB in, 4 GiB + 16 MiB + 12 bytes out, every
    output position past 2^32 - 1 and every match source inside the block's own output.  Run k and run k + 256 differ, so
    a decoder that wraps positions at 2^32 writes wrong bytes."""
    vals = [k % 251 + 1 for k in range(count)]
    tail = b"past 4 GiB!!"
    seqs = [Seq(bytes([v]), mlen, 1) for v in vals] + [Seq(tail)]
    return W.write_block(seqs), vals, tail
