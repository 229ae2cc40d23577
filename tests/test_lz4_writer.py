"""The hand-built LZ4 catalogue (tests/lz4_cases.py) on the CPU: the oracle answers every block, every frame and every cut as
the writer's model of the Swift decoder does, liblz4 decodes every valid block to the model's bytes, and the traces still
cover what the catalogue is for."""
import ctypes as C

import pytest

import helpers as H
import lz4_cases as D
import lz4_writer as W
from lz4_writer import Seq

F24 = 1 << 24


@pytest.fixture(scope="module")
def cases():
    return D.catalogue()


def test_canonical_block_matches_helpers():
    seqs = [(b"abcdefghijklmnopq", 19, 5), (b"", 4, 1), (b"x" * 300, 300, 200), (b"12", 274, 65535 - 400)]
    prefix = bytes(range(256)) * 300
    blk, raw = H.lz4_block_from_sequences(seqs, b"tail-literals", prefix)
    assert W.block(seqs, b"tail-literals") == blk
    r = W.decode_block(blk, prefix)
    assert r.status == W.OK and r.out == raw
    assert W.write_block([Seq(b"ab", 4, 1, lit_nib=15, lit_ext=b"\xFF\x00", off_raw=b"\x01", ml_nib=3)]) == b"\xF3\xFF\x00ab\x01"


def test_oracle_agrees_with_every_block(oracle, cases):
    bad = []
    for c in cases:
        if c.form != "block":
            continue
        st, out, _ = oracle.lz4_block(c.data, c.dictionary)
        if st != c.status or (st == W.OK and out != c.out):
            bad.append((c.name, st, c.status, len(out), len(c.out)))
    assert not bad, f"{len(bad)} of {len(cases)} cases differ from the oracle: {bad[:8]}"
    assert len(cases) > 900


def test_oracle_agrees_with_every_frame(oracle, cases):
    """family 8, and every block case wrapped as the single block of a dependent, an independent and a legacy frame"""
    bad, n = [], 0
    for c in cases:
        streams = [("frame", c.data, c.dictionary)] if c.form == "frame" else D.wrapped(c)
        for form, data, d in streams:
            n += 1
            m = W.decode(data, d)
            st, out, _ = oracle.lz4_decompress(data, d)
            if st != m.status or (st in (W.OK, W.CHECKSUM) and out != m.out):
                bad.append((c.name, form, st, m.status))
        if c.form == "frame":
            st, parts, _ = oracle.lz4_multi_decompress(c.data, c.dictionary)
            if (st, parts if st in (W.OK, W.CHECKSUM) else None) != (c.multi[0], c.multi[1] if st in (W.OK, W.CHECKSUM) else None):
                bad.append((c.name, "multi", st, c.multi[0]))
    assert not bad, f"{len(bad)} of {n} streams differ from the oracle: {bad[:8]}"
    assert n > 2000


def test_every_cut_decodes_as_the_model_says(oracle):
    cuts = D.truncations()
    assert len(cuts) > 5000
    bad = []
    for t in cuts:
        st, out, _ = oracle.lz4_block(t.data, t.case.dictionary)
        if st != t.model.status or out != t.model.out:
            bad.append((t.name, st, t.model.status, len(out), len(t.model.out)))
    assert not bad, f"{len(bad)} of {len(cuts)} cuts differ: {bad[:8]}"
    assert sum(t.model.status != W.OK for t in cuts) > 0.9 * len(cuts)


def test_liblz4_agrees(cases):
    """liblz4 owes nothing to the reference: every valid, non-empty block decodes with LZ4_decompress_safe_usingDict into
    exactly the model's bytes"""
    L = H.liblz4()
    fn = L.LZ4_decompress_safe_usingDict
    fn.restype = C.c_int
    fn.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_int]
    bad, n = [], 0
    for c in cases:
        if c.form != "block" or c.status != W.OK or not c.data:
            continue
        n += 1
        dst = C.create_string_buffer(max(len(c.out), 1))
        d = c.dictionary or b""
        got = fn(c.data, dst, len(c.data), len(c.out), d, len(d))
        if got != len(c.out) or dst.raw[:got] != c.out:
            bad.append((c.name, got, len(c.out)))
    assert not bad, f"liblz4 disagrees with {len(bad)} of {n} valid blocks: {bad[:8]}"
    assert n > 800


def test_coverage_contract(cases):
    """What the catalogue exists for, one assertion per item, so that an edit cannot quietly lose it"""
    blocks = [c for c in cases if c.form == "block"]
    trace = [e for c in blocks for e in c.model.trace]
    runs = {(e[1], e[2], e[3]) for e in trace if e[0] == "ext" and e[4]}
    for field in ("lit", "mlen"):
        assert {r for f, r, k in runs if f == field and r + k <= 32} == set(range(32)), f"{field} runs at every block residue"
        assert {r for f, r, k in runs if f == field and r + k > 32} == set(range(32)), f"{field} runs across a multiple of 32"
        assert {k for f, r, k in runs if f == field} >= set(range(1, 71)), f"{field} runs of 1..70 bytes"
        assert any(e[0] == "ext" and e[1] == field and not e[4] for e in trace), f"{field} run off the block"
    # the one-kernel decoder's window lanes (lane 1 cannot hold a match run: see lz4_cases.window_lanes)
    lanes = {(e[0], e[1], e[3]) for c in blocks for e in c.lanes}
    for field, reach in (("lit", set(range(32))), ("mlen", set(range(32)) - {1})):
        assert {l for f, l, x in lanes if f == field and not x} == reach, f"{field} runs inside the kernel window, every lane"
        assert {l for f, l, x in lanes if f == field and x} == reach, f"{field} runs across the kernel window, every lane"
    ok = [c for c in blocks if c.status == W.OK]
    lits = {e[2] for c in ok for e in c.model.trace if e[0] == "lit"}
    mlens = {e[4] for c in ok for e in c.model.trace if e[0] == "match"}
    assert set(range(17)) | {269, 270, 271, 524, 525, F24 - 1, F24} <= lits, "literal counts"
    assert set(range(4, 20)) | {273, 274, 528, 529, F24 - 1, F24} <= mlens, "match lengths"
    final = {c.model.trace[-1][2] for c in ok}
    assert {F24 - 1, F24} <= final, "final literal runs on both sides of 2^24"
    mixed = {c.name: c for c in ok}["lit_and_mlen_mixed"].model
    assert mixed.max_lit == F24 and mixed.max_mlen == F24 and mixed.nseq == 4
    matches = [e for c in ok for e in c.model.trace if e[0] == "match"]
    offs = {e[3] for e in matches}
    assert set(D.OFFSETS) <= offs, "offsets"
    assert {(e[3], e[4]) for e in matches if e[7]} >= {(o, m) for o in (1, 2, 3, 7, 16, 17, 32) for m in D.MLENS if o < m}
    assert {(e[5] == 0, c.dictionary is not None) for c in ok for e in c.model.trace if e[0] == "match"} >= \
        {(True, False), (True, True)}, "offset == out.endIndex, with and without a dictionary"
    rejected = {(e[1], c.dictionary is not None) for c in blocks for e in c.model.trace if e[0] == "offset"}
    assert {(1, False), (1, True)} <= rejected, "offset == out.endIndex + 1, with and without a dictionary"
    zero = [c for c in blocks if c.name.startswith("offset_0_op_")]
    assert len(zero) == 4 and all(c.model.trace[-1] == ("offset", -c.model.trace[-2][2]) for c in zero), "offset 0"
    kinds = {(e[6], e[7]) for e in matches}
    assert {("out", False), ("out", True), ("dict", False), ("dict", True), ("straddle", False), ("straddle", True)} <= kinds
    dicts = {len(c.dictionary) for c in ok if c.dictionary is not None and any(e[0] == "match" and e[6] != "out" for e in c.model.trace)}
    assert dicts == set(D.DICT_LENGTHS) - {0}, "sources in every non-empty dictionary"
    assert {len(c.dictionary) for c in blocks if c.dictionary is not None} == set(D.DICT_LENGTHS)
    ends = {e[1] for e in trace if e[0] == "end"}
    assert ends == {"single", "ok", "short_literals", "match_near_end"}, "every end rule"
    end_ok = {(e[2], e[3]) for c in ok for e in c.model.trace if e[0] == "end" and e[1] == "ok"}
    assert any(l == 5 for l, _ in end_ok) and any(d == 12 for _, d in end_ok), "final literal run 5, last match 12 from the end"
    end_bad = {(e[1], e[2], e[3]) for e in trace if e[0] == "end" and e[1] != "ok"}
    assert ("match_near_end", 5, 11) in end_bad and ("short_literals", 4, 11) in end_bad and ("short_literals", 4, 12) in end_bad
    assert {e[2] for e in trace if e[0] == "end" and e[1] == "single"} >= set(range(5)), "a lone sequence of 0..4 literals"
    assert {e[1] for e in trace if e[0] == "trunc"} == {"token", "lit_ext", "lits", "offset", "mlen_ext"}, "every cut kind"
    nseq = {c.model.nseq for c in ok}
    assert {31, 32, 33, 63, 64, 65} <= nseq, "record counts around the 32-record groups"
    dep = {e[1] for e in matches if e[8]}
    assert {r % 8 for r in dep} == set(range(8)), "a dependent match at every position of an 8-record batch"
    assert {8, 32, 64} <= dep, "a dependent match on the first record of a batch and of a group"
    long_then = [c for c in ok if c.name.startswith("long_match_at_")]
    for c in long_then:
        ms = [e for e in c.model.trace if e[0] == "match"]
        k = next(i for i, e in enumerate(ms) if e[4] == 100)
        start, end = ms[k][2], ms[k][2] + 100
        assert all(start <= e[2] - e[3] < end for e in ms[k + 1:]), c.name
    assert len(long_then) == 6
    edge = {e[1] for c in ok if c.name.startswith("literals_6") for e in c.model.trace if e[0] == "lit" and e[2] in (63, 64, 65)}
    assert edge == {7, 8, 31, 32}
    st = {c.name: c.status for c in cases}
    assert st["empty_block"] == W.TRUNCATED and st["ends_after_match"] == W.TRUNCATED
    frames = {c.name: c for c in cases if c.form == "frame"}
    assert {st[k] for k in ("chain_back_65535_from_stored_block", "chain_back_65535_across_two_blocks", "chain_into_stored_block", "chain_window_after_short_block",
                            "chain_zero_stored_then_dict", "chain_dict_first_block", "chain_dict_100000_window",
                            "independent_dict_each_block", "chain_empty_dict_present")} == {W.OK}
    assert {st[k] for k in ("chain_beyond_short_block", "chain_stored_then_dict_reach", "chain_dict_second_block_refused")} == {W.CORRUPTED}
    for nb in (1, 2, 33):
        for k in sorted({0, nb // 2, nb - 1}):
            assert st[f"chain_{nb}_fail_{k}_badck_none"] == W.TRUNCATED
            assert st[f"chain_{nb}_fail_{k}_badck_+0"] == W.CORRUPTED, "block k's checksum before its decode"
            if k > 0:
                assert st[f"chain_{nb}_fail_{k}_badck_-1"] == W.CORRUPTED
            if k + 1 < nb:
                assert st[f"chain_{nb}_fail_{k}_badck_+1"] == W.TRUNCATED, "block k's decode before block k + 1's checksum"
    assert len(frames["chain_33_fail_32_badck_-1"].model.blocks) == 31, "blocks 0..30 decode, block 31's checksum stops"
    assert st["chain_content_checksum_wrong"] == W.CHECKSUM and st["chain_content_size_wrong"] == W.CORRUPTED
    assert frames["multi_frames_with_dict"].multi[0] == W.OK and len(frames["multi_frames_with_dict"].multi[1]) == 3
    assert frames["multi_frames_truncated_last"].multi[0] == W.TRUNCATED


def test_past_4gib_block_shape(oracle):
    """the 4 GiB block of tests/test_gpu_lz4_handmade.py, scaled down: each sequence is one run of equal bytes"""
    blk, vals, tail = D.past_4gib_block(count=300, mlen=1000)
    want = b"".join(bytes([v]) * 1001 for v in vals) + tail
    assert W.decode_block(blk).out == want and oracle.lz4_block(blk)[:2] == (W.OK, want)
    blk, vals, _ = D.past_4gib_block()
    assert len(vals) == 257 and vals[0] != vals[256] and 16_000_000 < len(blk) < 17_000_000


def test_kernel_window_restatement():
    """W.kernel_window_runs on blocks whose window lanes follow from lz4.cu by hand"""
    lit_run = bytes([0xF4]) + b"\xFF\x00" + bytes(270) + b"\x01\x00" + bytes([0x00])
    assert W.kernel_window_runs(lit_run) == [("lit", 1, 2, False)]
    # 29 literals: the offset at 31-32 re-bases the window there, and the match run starts at lane 2 (never lane 1)
    blk = W.block([(bytes(29), 19 + 255 * 40, 1)], bytes(12))
    assert W.kernel_window_runs(blk)[-1] == ("mlen", 2, 41, True)
    # 28 literals: the offset fills lanes 30-31 and the match run opens the next window at lane 0
    blk = W.block([(bytes(28), 19, 1)], bytes(12))
    assert W.kernel_window_runs(blk) == [("lit", 1, 1, False), ("mlen", 0, 1, False)]
