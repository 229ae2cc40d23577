"""The hand-built LZMA / LZMA2 catalogue (tests/lzma_cases.py) on the CPU: the oracle answers every case as the writer's
model of the Swift decoder does (status, output, consumed bytes, and the output appended before a failure), liblzma agrees
with every case it can decode, every cut fails as the model says, and the traces still cover what the catalogue is for."""
import lzma

import pytest

import lzma_cases as D
import lzma_writer as W

MIB = 1 << 20


@pytest.fixture(scope="module")
def cases():
    return D.catalogue()


def oracle_answer(oracle, c, data=None):
    data = c.data if data is None else data
    if c.form == "raw":
        return oracle.lzma_decompress_raw(data, c.lc, c.lp, c.pb, c.dict_size, None if c.usize < 0 else c.usize)
    if c.form == "alone":
        return oracle.lzma_decompress(data)
    return oracle.lzma2_decompress_raw(data, c.dict_byte)


def model_answer(c, data):
    if c.form == "raw":
        return W.decode_lzma(data, c.lc, c.lp, c.pb, c.dict_size, c.usize)
    if c.form == "alone":
        return W.decode_lzma_alone(data)
    return W.decode_lzma2(data, c.dict_byte)


def test_oracle_agrees_with_every_case(oracle, cases):
    bad = []
    for c in cases:
        st, out, used = oracle_answer(oracle, c)
        if st != c.status:
            bad.append((c.name, st, c.status))
        elif c.unexpressible:
            continue
        elif out != c.model.out:
            bad.append((c.name, "output", len(out), len(c.model.out)))
        elif st != W.TRAP and used != c.model.consumed:            # a trap has no consumed count in the reference
            bad.append((c.name, "consumed", used, c.model.consumed))
    assert not bad, f"{len(bad)} of {len(cases)} cases differ from the oracle: {bad[:8]}"
    assert len(cases) > 700


def test_liblzma_agrees(cases):
    """liblzma owes nothing to the reference: the cases written in its subset (LZMA1 with lc + lp <= 4 and a dictionary of
    at least 4 KiB, LZMA2 whose first chunk resets the dictionary) must decode to the model's bytes"""
    bad, n = [], 0
    for c in cases:
        if not c.liblzma:
            continue
        n += 1
        if c.form == "raw":
            filt = {"id": lzma.FILTER_LZMA1, "lc": c.lc, "lp": c.lp, "pb": c.pb, "dict_size": c.dict_size}
        else:
            filt = {"id": lzma.FILTER_LZMA2, "dict_size": W.lzma2_dict_size(c.dict_byte)}
        d = lzma.LZMADecompressor(lzma.FORMAT_RAW, filters=[filt])
        try:
            out = d.decompress(c.data)
        except lzma.LZMAError as e:
            bad.append((c.name, str(e)))
            continue
        if out != c.model.out:
            bad.append((c.name, "bytes", len(out), len(c.model.out)))
    assert not bad, f"liblzma disagrees with {len(bad)} of {n} cases: {bad[:8]}"
    assert n >= 40


def test_every_cut_fails_as_the_model_says(oracle):
    cuts = D.truncations()
    assert len(cuts) > 20000
    bad = []
    for t in cuts:
        st, out, _ = oracle_answer(oracle, t.case, t.data)
        m = model_answer(t.case, t.data)
        if st == W.OK or st != m.status or out != m.out:
            bad.append((t.name, st, m.status, len(out), len(m.out)))
    assert not bad, f"{len(bad)} of {len(cuts)} cuts differ: {bad[:8]}"


def test_unexpressible_raw_properties(oracle, cases):
    """lc > 8, lp > 4 or pb > 4: the reference decodes lc = 9 (>> by -1 shifts left) and pb = 5 literals, and traps on a
    length at posState >= 16; the oracle and the engine refuse them all as UNSUPPORTED"""
    cat = {c.name: c for c in cases}
    want = {"raw_lc9_decodes": W.OK, "raw_lc9_lp4": W.OK, "raw_pb5_literals_decode": W.OK,
            "raw_pb5_match_at_posstate_17": W.TRAP, "raw_pb5_match_at_posstate_3": W.OK, "raw_lp5": W.OK}
    assert {k: cat[k].model.status for k in want} == want
    assert any(e[3][0] > 255 for e in cat["raw_lc9_lp4"].model.trace if e[0] == "lit"), "lc 9 reaches tables past 2^8"
    for k in want:
        assert cat[k].status == W.UNSUPPORTED and oracle_answer(oracle, cat[k])[0] == W.UNSUPPORTED


def test_lzma_properties_clamp_on_assignment_only():
    from swcompression_b200 import LZMAProperties
    p = LZMAProperties(lc=3, lp=0, pb=2, dictionarySize=1)
    assert p.dictionarySize == 1, "construction keeps any size (Swift's init does not call didSet)"
    p.dictionarySize = 0
    assert p.dictionarySize == 4096
    p.dictionarySize = 4095
    assert p.dictionarySize == 4096
    p.dictionarySize = 5000
    assert p.dictionarySize == 5000
    assert LZMAProperties().dictionarySize == 1 << 24 and LZMAProperties(dictionarySize=-1).dictionarySize == -1


def test_coverage_contract(cases):
    """What the catalogue exists for, one assertion per item, so that an edit cannot quietly lose it"""
    ok = [c for c in cases if c.status == W.OK]
    trace = [e for c in cases for e in c.model.trace]
    kinds = {"lit": "lit", "mlit": "lit", "match": "match", "rep0": "rep0", "rep1": "rep1", "rep2": "rep2", "rep3": "rep3",
             "short": "short", "end": "end"}
    sk = {(e[1], kinds[e[0]]) for e in trace}
    assert {(s, k) for s in range(12) for k in set(kinds.values())} <= sk, "every (state, symbol kind)"
    slots = {e[3][2] for e in trace if e[0] in ("match", "end")}
    assert set(range(64)) <= slots, "every pos slot"
    real = {e[3][2] for c in ok for e in c.model.trace if e[0] == "match"}
    assert set(range(46)) <= real, "slots 0..45 as decoded matches"
    assert max(len(c.model.out) for c in ok) >= 8 * MIB
    vals = {(e[3][2], e[3][3] - D.slot_base(e[3][2])) for e in trace if e[0] == "match" and 4 <= e[3][2] < 14}
    assert all((s, r) in vals for s in range(4, 14) for r in range(1 << ((s >> 1) - 1))), "every reverse-tree value, slots 4..13"
    align = {(e[3][3] - 128) & 15 for e in trace if e[0] == "match" and e[3][2] == 14}
    assert align == set(range(16)), "every align value"
    pb4 = [c for c in cases if c.family == 4]
    for coder, k in (("match", "match"), ("rep", "rep1")):
        got = {(e[2], e[3][1]) for c in pb4 for e in c.model.trace if e[0] == k}
        assert {(ps, L) for ps in range(16) for L in range(272)} <= got, f"{coder} lengths 2..273 at every posState"
    branches = {(e[2], e[3][0]) for c in pb4 for e in c.model.trace if e[0] in ("match", "rep1")}
    assert {(ps, b) for ps in range(16) for b in ("low", "mid", "high")} <= branches, "both coders' branches per posState"
    tables = {e[3][0] for c in cases if (c.lc, c.lp) == (8, 4) or c.form == "alone" and c.data[0] == 8 + 9 * 4
              for e in c.model.trace if e[0] in ("lit", "mlit")}
    assert 4095 in tables, "literal table 4095 at lc 8, lp 4"
    lcs = {(c.data[0] % 9, (c.data[0] // 9) % 5) for c in ok if c.form == "alone"}
    assert {(lc, lp) for lc in range(9) for lp in range(5)} <= lcs, "every lc, lp through a header"
    left = {e[3][1] for e in trace if e[0] == "mlit"}
    assert set(range(8)) | {None} <= left, "matched literals leaving the match byte at each bit, and not at all"
    assert any(c.name == "state_11_posstate_15_short" and c.model.status == W.TRAP for c in cases), "isRep0Long entry 432"
    st = {c.name: c.model.status for c in cases}
    assert st["dict_1_literals"] == W.OK and st["dict_1_rep0_after_literals"] == W.WINDOW_EMPTY
    assert {st["dict_4096_match_at_size_minus_1"], st["dict_4096_match_at_size"]} == {W.OK, W.NOT_ENOUGH}, "dictSize - 1 / dictSize"
    assert st["dict_4096_match_at_dict_end"] == W.TRAP, "rep0 == dictEnd < dictSize traps in byte(at:)"
    one = {e[3][0] for c in cases if c.name == "dict_1_literals" for e in c.model.trace}
    assert one == {0}, "a 1-byte dictionary keeps every literal at context 0"
    for k in ("size_reached_then_literal", "size_reached_then_rep", "size_reached_then_short"):
        assert st[k] == W.EXCEEDED, k
    assert st["size_reached_then_end"] == W.OK and st["end_marker_before_size"] == W.OK
    assert st["end_marker_then_literal"] == W.FINISH_ERROR and st["match_longer_than_left"] == W.REPEAT_EXCEED
    assert st["first_byte_1"] == W.INIT_ERROR and st["input_4_bytes"] == W.INIT_ERROR
    controls = {c.data[o] for c in cases if c.form == "lzma2" for o in c.model.controls if o < len(c.data)}
    assert {0, 1, 2, 3, 0x7F} | {0x80, 0xA0, 0xC0, 0xE0} <= {b if b < 0x80 else b & 0xE0 for b in controls}, "every control class"
    assert st["l2_reset0_first_traps"] == W.TRAP and st["l2_reset1_first_defaults"] == W.OK
    assert st["l2_dict_reset_chunk_rep"] == W.WINDOW_EMPTY and st["l2_dict_reset_chunk_match_behind"] == W.OK
    assert {st["l2_unpack_too_large"], st["l2_comp_plus_1"], st["l2_comp_minus_1"]} == {W.WRONG_SIZES}, "wrongSizes from each field"
    assert {st[f"l2_dict_byte_{b}"] for b in range(40)} == {W.OK} and {st[f"l2_dict_byte_{b}"] for b in (40, 63, 64, 128)} == {W.WRONG_DICT}
    big = [c for c in ok if c.form == "lzma2"]
    assert max(len(c.model.out) for c in big) == 2 * MIB and max(len(c.data) for c in big) > 64000, "2 MiB / 64 KiB chunks"
    res = {o % 128 for c in cases if c.family == 8 for o in c.model.controls} | {len(c.data) % 128 for c in cases if c.family == 8}
    assert {0, 1, 126, 127} <= res, "chunk boundaries and stream ends at residues 0, 1, 126, 127 of 128"
    assert sum(c.batch == W.UNSUPPORTED and not c.unexpressible for c in cases) >= 2 * 9 * 5
