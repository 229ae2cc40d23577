"""The hand-built LZMA / LZMA2 catalogue (tests/lzma_cases.py) on lzma_kernel, unit by unit against the oracle.  The units
are packed the hostile way of tests/test_gpu_layout.py and run at capacities of exactly the decoded size and one byte
short; statuses are compared exactly, the batched forms answering UNSUPPORTED once a unit reaches lc + lp > 4 (DESIGN §6).
A failing unit gets exactly the bytes the oracle appends before it fails: it must fail as the oracle does, with the same
out_len and bytes, and with one byte less it must report OVERFLOW.

The single-stream API runs every case (literal coders in global scratch for lc + lp > 4, the x4 capacity retry), XZ
archives mix lc + lp > 4 blocks with ordinary ones (the prefetch batch and the in-order fallback), and a ZIP container
holds an lc = 8, lp = 4 LZMA entry among ordinary ones."""
import io
import struct
import zipfile
import zlib

import numpy as np
import pytest

import helpers as H
import lzma_cases as D
import lzma_writer as W
from test_gpu_layout import Layout, run_both, run_lzma, run_lzma2

pytestmark = pytest.mark.gpu


def _units(cases):
    """-> (raw LZMA units with their (props, dict size, size) and batch statuses, LZMA2 units and batch statuses)"""
    raw, raw_st, l2, l2_st = [], [], [], []
    for c in cases:
        if c.form == "lzma2":
            l2.append(H.LayoutUnit(c.data, aux=c.dict_byte, raw=c.model.out if c.status == 0 else None))
            l2_st.append(c.batch)
            continue
        if c.form == "alone":
            b = c.data[0]
            if b >= 225:
                continue
            props = b % 9 | ((b // 9) % 5) << 8 | (b // 45) << 16
            aux = (props, int.from_bytes(c.data[1:5], "little"), max(int.from_bytes(c.data[5:13], "little", signed=True), -1))
            data = c.data[13:]
        else:
            aux, data = (c.props, c.dict_size, c.usize), c.data
        raw.append(H.LayoutUnit(data, aux=aux, raw=c.model.out if c.status == 0 else None))
        raw_st.append(c.batch)
    return raw, raw_st, l2, l2_st


def _caps(lay, short):
    """every unit's output region: the oracle's output length (a failing unit's appended bytes) minus `short`"""
    offs = np.zeros(lay.n, dtype=np.uint64)
    caps = np.zeros(lay.n, dtype=np.uint64)
    pos = H.GUARD
    for i, e in enumerate(lay.expect):
        cap = max(len(e[1]) - short, 0)
        offs[i], caps[i] = pos, cap
        pos = (pos + cap + 1 + 15) // 16 * 16
    lay.out_off, lay.out_cap, lay.total = offs, caps, pos + H.GUARD


def _check_failures(lay, engine, st, ln, out):
    """failing units at the oracle's appended size: the oracle's status, out_len and bytes"""
    bad = []
    for i, (ost, oout, _) in enumerate(lay.expect):
        o = int(lay.out_off[i])
        if ost != 0 and engine[i] == ost and (st[i] != ost or ln[i] != len(oout) or bytes(out[o:o + len(oout)]) != oout):
            bad.append((i, int(st[i]), ost, int(ln[i]), len(oout)))
    assert not bad, f"{len(bad)} failing units differ: {bad[:8]}"


def _short(lay, engine):
    """one byte below the oracle's output a failing unit overflows before it reaches its error"""
    return [W.OVERFLOW if e[0] != 0 and s == e[0] and e[1] else s for e, s in zip(lay.expect, engine)]


def _run(codec, units, engine, run, seed, oracle):
    lay = Layout(codec, oracle, units, seed)
    _caps(lay, 0)
    st, ln, used, out = run_both(lay, run)
    lay.check(st, ln, used, out, engine=engine)
    _check_failures(lay, engine, st, ln, out)
    _caps(lay, 1)
    lay.check(*run_both(lay, run), engine=_short(lay, engine))
    return lay


def test_catalogue_batch(oracle):
    cases = D.catalogue()
    raw, raw_st, l2, l2_st = _units(cases)
    lay = _run("lzma", raw, raw_st, run_lzma, 501, oracle)
    assert sum(e[0] != 0 for e in lay.expect) > 50
    lay = _run("lzma2", l2, l2_st, run_lzma2, 502, oracle)
    assert sum(s == W.UNSUPPORTED for s in raw_st + l2_st) >= 90


def test_truncations_batch(oracle):
    cuts = D.truncations()
    raw, raw_st, l2, l2_st = [], [], [], []
    for t in cuts:
        c = t.case
        if c.form == "lzma2":
            l2.append(H.LayoutUnit(t.data, tail=t.tail, aux=c.dict_byte))
            l2_st.append(W.decode_lzma2(t.data, c.dict_byte).batch_status())
        elif c.form == "raw":
            raw.append(H.LayoutUnit(t.data, tail=t.tail, aux=(c.props, c.dict_size, c.usize)))
            raw_st.append(c.batch if c.unexpressible else
                          W.decode_lzma(t.data, c.lc, c.lp, c.pb, c.dict_size, c.usize).batch_status())
    assert len(raw) + len(l2) > 7000
    for codec, units, engine, run, seed in (("lzma", raw, raw_st, run_lzma, 503), ("lzma2", l2, l2_st, run_lzma2, 504)):
        lay = Layout(codec, oracle, units, seed)
        assert all(e[0] != 0 for e in lay.expect)
        _caps(lay, 0)
        st, ln, used, out = run_both(lay, run)
        lay.check(st, ln, used, out, engine=engine)
        _check_failures(lay, engine, st, ln, out)


def test_single_stream_api():
    """LZMA.decompress (header and raw forms) and LZMA2.decompress on every case"""
    import swcompression_b200 as S
    bad = []
    for c in D.catalogue():
        try:
            if c.form == "alone":
                got = (0, S.LZMA.decompress(c.data))
            elif c.form == "raw":
                p = S.LZMAProperties(lc=c.lc, lp=c.lp, pb=c.pb, dictionarySize=c.dict_size)
                got = (0, S.LZMA.decompress(c.data, p, None if c.usize < 0 else c.usize))
            else:
                got = (0, S.LZMA2.decompress(bytes([c.dict_byte]) + c.data))
        except S.SWCompressionError as e:
            got = (e.code, None)
        want = (c.status, c.model.out if c.status == 0 else None)
        if got != want:
            bad.append((c.name, got[0], want[0]))
    assert not bad, f"{len(bad)} cases differ: {bad[:8]}"


def _xz(blocks):
    """an XZ stream without checks whose blocks are (LZMA2 stream with its end byte, dictionary byte)"""
    import test_framing_handmade as F
    body, recs = b"", []
    for data, db, size in blocks:
        blk, unpadded = F.xz_block(check=0, filt=b"\x21\x01" + bytes([db]), data=data, check_bytes=b"")
        body += blk
        recs.append((unpadded, size))
    idx = F.xz_index(recs)
    return F.xz_header(0) + body + idx + F.xz_footer(len(idx), 0)


def test_xz_mixes_wide_literal_blocks():
    """blocks with lc + lp > 4 are refused by the prefetch batch and decoded by the in-order parser; ordinary blocks around
    them come from the batch"""
    import swcompression_b200 as S
    cat = {c.name: c for c in D.catalogue()}
    wide = [cat["l2_props_lc8_lp4"], cat["l2_props_lc4_lp1_after_small"]]
    plain = [cat["l2_reset3_first"], cat["l2_stored1_first"], cat["l2_chunk_2_mib_unpacked"]]
    assert all(c.batch == W.UNSUPPORTED and c.status == 0 for c in wide) and all(c.batch == 0 for c in plain)
    for order in ([plain[0], wide[0], plain[1]], [wide[0], wide[1]], [plain[2], wide[1], plain[0], wide[0]], plain[:2]):
        arch = _xz([(c.data, c.dict_byte, len(c.model.out)) for c in order])
        assert S.XZArchive.unarchive(arch) == b"".join(c.model.out for c in order)
    two = _xz([(c.data, c.dict_byte, len(c.model.out)) for c in (plain[0], wide[0])])
    assert S.XZArchive.splitUnarchive(two + two) == [b"".join(c.model.out for c in (plain[0], wide[0]))] * 2


def _zip_with_lzma_entry(ordinary, name, payload, raw):
    """a ZIP container of `ordinary` entries and one LZMA entry (method 14) whose data is `payload`, patched into a stored one"""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w") as z:
        for n, d, m in ordinary[:2]:
            z.writestr(zipfile.ZipInfo(n, date_time=(2021, 3, 4, 5, 6, 8)), d, compress_type=m)
        z.writestr(zipfile.ZipInfo(name, date_time=(2021, 3, 4, 5, 6, 8)), payload, compress_type=zipfile.ZIP_STORED)
        for n, d, m in ordinary[2:]:
            z.writestr(zipfile.ZipInfo(n, date_time=(2021, 3, 4, 5, 6, 8)), d, compress_type=m)
    b = bytearray(buf.getvalue())
    crc = zlib.crc32(raw)
    for sig, meth, crc_at, usize_at, name_len_at, head in ((b"PK\x03\x04", 8, 14, 22, 26, 30), (b"PK\x01\x02", 10, 16, 24, 28, 46)):
        p = b.find(sig)
        while p >= 0:
            nlen = struct.unpack_from("<H", b, p + name_len_at)[0]
            if bytes(b[p + head:p + head + nlen]) == name.encode():
                struct.pack_into("<H", b, p + meth, 14)
                struct.pack_into("<I", b, p + crc_at, crc)
                struct.pack_into("<I", b, p + usize_at, len(raw))
            p = b.find(sig, p + 4)
    return bytes(b)


def test_zip_lzma_entry_lc8_lp4(oracle):
    """the batch refuses the entry (lc + lp > 4) and the container decodes it again on its own"""
    import swcompression_b200 as S
    ops = D.lits(b"\xFF" * 32 + D.text(3000, 8000)) + [W.match(200, 1000), W.rep(0, 50)] + D.lits(b"tail")
    stream = W.write_lzma(ops, lc=8, lp=4, pb=4, dict_size=1 << 16)
    props = W.props_byte(8, 4, 4)
    raw = W.decode_lzma(stream, 8, 4, 4, 1 << 16, 32 + 3000 + 200 + 50 + 4)
    assert raw.status == 0 and len(raw.out) == 3286
    payload = b"\x09\x14\x05\x00" + bytes([props]) + (1 << 16).to_bytes(4, "little") + stream
    ordinary = [("a.txt", H.textlike(5000, 8001), zipfile.ZIP_DEFLATED), ("b.bin", H.textlike(20000, 8002), zipfile.ZIP_LZMA),
                ("c.txt", H.textlike(7000, 8003), zipfile.ZIP_LZMA), ("d.bz", H.textlike(3000, 8004), zipfile.ZIP_BZIP2)]
    blob = _zip_with_lzma_entry(ordinary, "wide.lzma", payload, raw.out)
    st, ents = oracle.zip_open(blob)
    assert st == 0
    got = S.ZipContainer.open(blob)
    assert [g.data for g in got] == [e["data"] for e in ents]
    assert [g.data for g in got] == [ordinary[0][1], ordinary[1][1], raw.out, ordinary[2][1], ordinary[3][1]]
