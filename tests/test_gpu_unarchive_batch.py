"""The batched unarchive calls (swc_gzip_unarchive_batch, swc_zlib_unarchive_batch) and swc_adler32_batch against the oracle's
gzip_unarchive / zlib_unarchive, the single-archive calls and the raw Deflate batch: status, output length, consumed bytes and
output bytes unit by unit (bytes on OK and on the payload-carrying statuses), on the catalogue of tests/unarchive_cases.py,
truncations, both Huffman stages, hostile layouts, output overflow and a CUDA-graph capture."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

import helpers as H
import unarchive_cases as U

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def S():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _expect(oracle, fmt, datas):
    cache, out = {}, []
    for d in datas:
        if d not in cache:
            cache[d] = U.oracle_unarchive(oracle, fmt, d)
        out.append(cache[d])
    return out


def _caps(expect, spare=None):
    sizes = [len(o) for st, o, _ in expect]
    spare = spare if spare is not None else max(sizes + [0]) + 4096
    return np.array([len(o) if st in (U.OK,) + U.PAYLOAD_CARRYING else spare for st, o, _ in expect], dtype=np.uint64)


def _header_fails(fmt, data):
    """the archive fails before its Deflate stream: gzip's 20-byte guard or the header grammar (host parse)"""
    from swcompression_b200 import _lib
    from swcompression_b200.api import _CGzipHeader, _CZlibHeader
    buf, n = _lib.inbuf(data)
    if fmt == "gzip":
        return n < 20 or _lib.lib().swc_gzip_header_parse(buf, n, 0, C.byref(_CGzipHeader())) != 0
    return _lib.lib().swc_zlib_header_parse(buf, n, C.byref(_CZlibHeader())) != 0


def _compare(fmt, datas, expect, st, ln, used, outs, caps=None):
    """unit-by-unit comparison with the oracle -> list of differences"""
    bad = []
    for i, (d, (ost, oout, oused)) in enumerate(zip(datas, expect)):
        carries = ost in (U.OK,) + U.PAYLOAD_CARRYING
        if carries and caps is not None and len(oout) > caps[i]:
            if st[i] != 1 or ln[i] != len(oout):
                bad.append((i, "overflow", int(st[i]), int(ln[i]), len(oout)))
            continue
        if st[i] != ost:
            bad.append((i, "status", int(st[i]), ost))
        elif carries and (ln[i] != len(oout) or outs[i][:len(oout)] != oout or used[i] != oused):
            bad.append((i, "payload/consumed", int(ln[i]), len(oout), int(used[i]), oused))
        elif not carries and used[i] != 0:
            bad.append((i, "consumed of a failed unit", int(used[i])))
        elif not carries and ln[i] != 0 and _header_fails(fmt, d):
            bad.append((i, "out_len of a header failure", int(ln[i])))
    return bad


def _run(fmt, datas, caps, headers=False):
    from swcompression_b200.batch import Batch
    b = Batch.from_units(fmt, datas, caps, headers=headers)
    b.run()
    st, ln, used = b.results()
    outs = b.outputs()
    return b, st, ln, used, outs


def _single_status(fmt, data):
    from swcompression_b200 import _lib
    L = _lib.lib()
    buf, n = _lib.inbuf(data)
    out, ol, used = C.c_void_p(), C.c_size_t(), C.c_size_t()
    if fmt == "gzip":
        st = L.swc_gzip_unarchive(buf, n, C.byref(out), C.byref(ol), C.byref(used))
    else:
        st = L.swc_zlib_unarchive(buf, n, C.byref(out), C.byref(ol))
    _lib.take(out, ol)
    return st


def test_golden_fixtures(S):
    """GZip/*.gz and the two zlib fixtures in one batch each give the single calls' answers and statuses"""
    rels = [rel for rel, _ in H.fixtures("GZip/")]
    datas = [H.fixture(r) for r in rels]
    _, st, ln, used, outs = _run("gzip", datas, 1 << 21)
    for i, (rel, ans) in enumerate(H.fixtures("GZip/")):
        assert st[i] == 0 and outs[i] == H.answer(ans) == S.GzipArchive.unarchive(datas[i]) and used[i] == len(datas[i]), rel
    zd = [H.fixture("Zlib/test_empty.zlib"), H.fixture("Zlib/test.zlib")]
    _, st, ln, used, outs = _run("zlib", zd, 1 << 21)
    assert st[0] == 0 and outs[0] == S.ZlibArchive.unarchive(zd[0]) == b"" and used[0] == len(zd[0])
    with pytest.raises(S.DeflateError) as e:
        S.ZlibArchive.unarchive(zd[1])
    assert st[1] == e.value.code == U.WRONG_BLOCK_TYPE and used[1] == 0


@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_catalogue(S, oracle, fmt):
    """every archive of unarchive_cases (header catalogue, trailer cases, the Deflate catalogue wrapped, Python's gzip / zlib at
    levels 0-9 with every optional header field) as one batch"""
    arcs = [a for a in U.cases() if a.fmt == fmt]
    datas = [a.data for a in arcs]
    expect = _expect(oracle, fmt, datas)
    caps = _caps(expect)
    b, st, ln, used, outs = _run(fmt, datas, caps, headers=True)
    bad = _compare(fmt, datas, expect, st, ln, used, outs)
    assert not bad, f"{len(bad)} of {len(arcs)} differ: {[(arcs[x[0]].name,) + x[1:] for x in bad[:8]]}"
    for a, s in zip(arcs, st):
        if a.status is not None:
            assert s == a.status, a.name
    # the header catalogue: the same status as the single-archive call, and (gzip) the header array as swc_gzip_header_parse
    from swcompression_b200 import _lib
    from swcompression_b200.api import _CGzipHeader
    hdrs = b.gzip_headers() if fmt == "gzip" else None
    offs = b.d_in_off.cpu().numpy().view(np.uint64)
    for i, a in enumerate(arcs):
        if not a.name.startswith(f"{fmt} header "):
            continue
        assert st[i] == _single_status(fmt, a.data), a.name
        if fmt != "gzip":
            continue
        h = _CGzipHeader()
        buf, n = _lib.inbuf(a.data)
        hst = _lib.lib().swc_gzip_header_parse(buf, n, 0, C.byref(h)) if len(a.data) >= 20 else U.GZ_MAGIC
        got = hdrs[i]
        if hst != 0:
            assert bytes(got) == bytes(_CGzipHeader()), a.name
            continue
        o = int(offs[i])
        if h.has_file_name:
            h.file_name_off += o
        if h.has_comment:
            h.comment_off += o
        if h.extra_len:
            h.extra_off += o
        for f, _ in _CGzipHeader._fields_:
            assert getattr(got, f) == getattr(h, f), (a.name, f)


@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_deflate_errors_inside_members_match_the_raw_batch(S, oracle, fmt):
    """the Deflate catalogue's bit-0 streams and streams with damaged dynamic headers (incomplete and over-subscribed code
    sets, which the slow kernel takes) inside members: wherever the bare stream (the archive behind its header) fails in the
    raw Deflate batch, the member fails with that status and output length"""
    from swcompression_b200.batch import Batch
    arcs = [a for a in U.deflate_member_cases() if a.fmt == fmt]
    head, trailer = (U.GZIP_HEAD, bytes(8)) if fmt == "gzip" else (U.ZLIB_HEAD, bytes(4))
    datas = [a.data for a in arcs] + [head + u.data + trailer for u in H.layout_malformed_deflate(random.Random(71), 80)]
    expect = _expect(oracle, fmt, datas)
    caps = _caps(expect)
    raw = Batch.from_units("deflate", [d[len(head):] for d in datas], caps)
    raw.run()
    rst, rln, _ = raw.results()
    _, st, ln, used, outs = _run(fmt, datas, caps)
    assert not _compare(fmt, datas, expect, st, ln, used, outs)
    failing = np.nonzero(rst != 0)[0]
    assert failing.size >= 30
    assert (st[failing] == rst[failing]).all() and (ln[failing] == rln[failing]).all()
    assert all(st[i] == a.status for i, a in enumerate(arcs) if a.status not in (None, U.OK))


def _truncations(rng):
    small = [U.gzip_member(H.textlike(150, 61), name=b"a.txt", flags=0x02), U.gzip_member(b"x" * 40, 0),
             U.zlib_stream(H.textlike(150, 62)), U.zlib_stream(b"", 0), U.gzip_member(b"")]
    large = [U.gzip_member(H.textlike(70000, 63), comment=b"big"), U.zlib_stream(H.textlike(90000, 64), 9)]
    cuts = []
    for a in small:
        cuts += [(a, k) for k in range(len(a) + 1)]
    for a in large:
        cuts += [(a, rng.randrange(len(a) + 1)) for _ in range(60)] + [(a, len(a) - k) for k in range(10)]
    return cuts


def test_truncations(S, oracle):
    """every cut of small archives and random cuts of large ones, the rest of the archive lying behind the unit in memory"""
    cuts = _truncations(random.Random(60))
    for fmt in ("gzip", "zlib"):
        mine = [(a, k) for a, k in cuts if (a[:2] == b"\x1f\x8b") == (fmt == "gzip")]
        datas = [a[:k] for a, k in mine]
        expect = _expect(oracle, fmt, datas)
        _, st, ln, used, outs = _run(fmt, datas, _caps(expect))
        bad = _compare(fmt, datas, expect, st, ln, used, outs)
        assert not bad, (fmt, bad[:8])


def test_both_huffman_stages(S, oracle):
    """fewer than 20 000 units take the warp decoder, 20 000 and more the table-lookup decoder: the same answers"""
    rng = random.Random(65)
    base = []
    for j in range(64):
        raw = H.textlike(rng.randrange(0, 3000), 650 + j)
        a = bytearray(U.gzip_member(raw, rng.choice([1, 6, 9]), name=b"u%d" % j if j % 4 == 0 else None))
        if j % 8 == 3:
            a[-6] ^= 1                                          # CRC
        elif j % 8 == 5:
            a = a[:len(a) // 2]                                 # cut
        base.append(bytes(a))
    for n in (19999, 20480):
        datas = [base[i % 64] for i in range(n)]
        expect = _expect(oracle, "gzip", datas)
        _, st, ln, used, outs = _run("gzip", datas, _caps(expect, 4096))
        bad = _compare("gzip", datas, expect, st, ln, used, outs)
        assert not bad, (n, bad[:8])


@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_hostile_layout(S, oracle, fmt):
    """unaligned and back-to-back units, cut archives followed by their own rest, output regions of every capacity residue
    (exact, 1-15 bytes short: overflow with the size required, 1-15 long) inside sentinel bytes that must stay intact; then
    one unit alone, followed by another member's start, in a region far larger than its output (a one-unit batch spreads
    its checksum over the whole region)"""
    import torch
    from swcompression_b200 import _lib
    rng = random.Random(66 if fmt == "gzip" else 67)
    make = U.gzip_member if fmt == "gzip" else U.zlib_stream
    units, tails = [], []
    for j in range(90):
        raw = H.textlike(rng.choice([0, 1, 100, 3000, 20000]), 670 + j) if j % 5 else H.random_bytes(rng, rng.randrange(0, 2000))
        a = U.gzip_member(raw, rng.choice([0, 1, 6, 9]), name=b"h" if j % 3 == 0 else None) if fmt == "gzip" else \
            U.zlib_stream(raw, rng.choice([0, 1, 6, 9]))
        if j % 4 == 1:
            c = rng.randrange(1, len(a))
            units.append(a[:c]); tails.append(a[c:])
        elif j % 4 == 2:
            b = bytearray(a); b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            units.append(bytes(b)); tails.append(None)
        else:
            units.append(a); tails.append(b"\x1f\x8b\x08\x00" if j % 2 else None)
    L = _lib.lib()
    for units, tails, alone in ((units, tails, False), ([make(H.textlike(100000, 669))], [b"\x1f\x8b\x08\x00"], True)):
        expect = _expect(oracle, fmt, units)
        sizes = [len(o) if s in (U.OK,) + U.PAYLOAD_CARRYING else None for s, o, _ in expect]
        spare = max(len(o) for _, o, _ in expect) + 1024      # a failing unit stops at its error, within what the oracle wrote
        out_off, out_cap, total = H.fenced_layout([None] if alone else sizes, 40 * spare if alone else spare)
        buf, offs, lens = H.pack_hostile(units, rng, None, tails)
        n = len(units)
        d_in, d_off, d_len, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
        d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
        d_ln, d_used = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda")
        d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        scratch = torch.empty(L.swc_unarchive_batch_scratch_bytes(n, total), dtype=torch.uint8, device="cuda")
        args = [_p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_oo), _p(d_oc), total, _p(d_ln), _p(d_used), _p(d_st)]
        if fmt == "gzip":
            st = L.swc_gzip_unarchive_batch(*args, None, n, _p(scratch), scratch.numel(), _stream())
        else:
            st = L.swc_zlib_unarchive_batch(*args, n, _p(scratch), scratch.numel(), _stream())
        assert st == 0
        torch.cuda.synchronize()
        out = d_out.cpu().numpy()
        stv, lnv, usedv = d_st.cpu().numpy(), d_ln.cpu().numpy(), d_used.cpu().numpy()
        outs = [bytes(out[int(o):int(o) + int(c)]) for o, c in zip(out_off, out_cap)]
        bad = _compare(fmt, units, expect, stv, lnv, usedv, outs, caps=out_cap)
        fence = H.fence_violations(out, out_off, out_cap)
        assert not bad and fence.size == 0, (alone, bad[:8], fence[:8])
        assert (stv == 0).all() if alone else (stv == 1).sum() > 5


def test_output_overflow_then_rerun(S):
    """a capacity below ISIZE reports SWC_ERR_OUTPUT_OVERFLOW with the size required; a rerun at that size decodes"""
    raws = [H.textlike(n, 680 + n) for n in (1, 100, 5000, 65536)]
    for fmt, make in (("gzip", U.gzip_member), ("zlib", U.zlib_stream)):
        datas = [make(r) for r in raws]
        _, st, ln, _, _ = _run(fmt, datas, np.array([len(r) - 1 for r in raws], dtype=np.uint64))
        assert (st == 1).all() and list(ln) == [len(r) for r in raws]
        _, st, ln, used, outs = _run(fmt, datas, ln.astype(np.uint64))
        assert (st == 0).all() and outs == raws and list(used) == [len(d) for d in datas]


def test_adler32_batch(S):
    """swc_adler32_batch equals zlib.adler32 for every length 0-64, around 5 552 and 2^20, random and all-0xFF bytes, at
    every start alignment; units whose status is not 0 are skipped and left at 0"""
    import torch
    from swcompression_b200 import _lib
    rng = random.Random(69)
    lens = list(range(65)) + list(range(5540, 5566)) + [(1 << 20) + d for d in (-17, -1, 0, 1, 16)]
    units = []
    for n in lens:
        units.append(H.random_bytes(rng, n) if n < 6000 else np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes())
        units.append(b"\xff" * n)
    buf, offs, ulens = H.pack_hostile(units, rng)
    n = len(units)
    status = np.zeros(n, dtype=np.int32)
    status[7::11] = 605
    d_buf, d_off, d_len, d_st = _dev(buf), _dev(offs), _dev(ulens), _dev(status)
    d_res = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    assert L.swc_adler32_batch(_p(d_buf), _p(d_off), _p(d_len), _p(d_st), _p(d_res), n, _stream()) == 0
    assert L.swc_adler32_batch(_p(d_buf), _p(d_off), _p(d_len), None, None, n, _stream()) == 4
    torch.cuda.synchronize()
    got = d_res.cpu().numpy().view(np.uint32)
    want = [0 if status[i] else zlib.adler32(u) for i, u in enumerate(units)]
    bad = [(i, len(units[i]), int(got[i]), want[i]) for i in range(n) if got[i] != want[i]]
    assert not bad, bad[:8]


def test_invalid_arguments(S):
    import torch
    from swcompression_b200 import _lib
    L = _lib.lib()
    datas = [U.zlib_stream(b"abc")]
    from swcompression_b200.batch import Batch
    b = Batch.from_units("zlib", datas, 16)
    p = lambda t: C.c_void_p(t.data_ptr())
    args = [p(b.d_in), p(b.d_in_off), p(b.d_in_len), p(b.d_out), p(b.d_out_off), p(b.d_out_cap), b.out_total, p(b.d_out_len),
            p(b.d_consumed), p(b.d_status)]
    need = L.swc_unarchive_batch_scratch_bytes(1, b.out_total)
    assert L.swc_zlib_unarchive_batch(*args, 1, p(b.d_scratch), need - 1, _stream()) == 4
    assert L.swc_zlib_unarchive_batch(*args[:9], None, 1, p(b.d_scratch), need, _stream()) == 4
    assert L.swc_zlib_unarchive_batch(*args, 0, None, 0, _stream()) == 0
    assert L.swc_zlib_unarchive_batch(*args, 1, None, 0, _stream()) == 0          # library pool
    torch.cuda.synchronize()
    assert b.results()[0][0] == 0 and b.outputs()[0] == b"abc"


@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_graph_capture(S, oracle, fmt):
    """with caller scratch the call is one enqueue: after an eager warm-up it is captured into a CUDA graph and the replay
    gives the eager results (no host synchronisation or allocation on the path), for a batch of 200 units and for one unit
    whose capacity is far above its output (the one-unit checksum path)"""
    import torch
    rng = random.Random(70)
    make = (lambda raw: U.gzip_member(raw, name=b"g")) if fmt == "gzip" else U.zlib_stream
    datas = []
    for j in range(200):
        raw = H.textlike(rng.randrange(0, 8000), 700 + j)
        a = bytearray(make(raw))
        if j % 7 == 3:
            a[-2] ^= 4
        datas.append(bytes(a[:len(a) - 3] if j % 11 == 5 else a))
    one = make(H.textlike(300000, 699))
    from swcompression_b200.batch import Batch
    for datas, caps in ((datas, None), ([one], np.array([64 * len(one)], dtype=np.uint64))):
        expect = _expect(oracle, fmt, datas)
        b = Batch.from_units(fmt, datas, _caps(expect) if caps is None else caps, headers=True)
        b.run()
        st0, ln0, used0 = b.results()
        outs0 = b.outputs()
        assert not _compare(fmt, datas, expect, st0, ln0, used0, outs0)
        h0 = b.d_headers.clone() if b.d_headers is not None else None
        b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_consumed.zero_(); b.d_out.zero_()
        if h0 is not None:
            b.d_headers.zero_()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                b.run()
        torch.cuda.synchronize()
        assert (b.d_status.cpu().numpy() == -1).all()          # captured, not run
        g.replay()
        st1, ln1, used1 = b.results()
        assert (st1 == st0).all() and (ln1 == ln0).all() and (used1 == used0).all() and b.outputs() == outs0
        if h0 is not None:
            assert torch.equal(b.d_headers, h0)
