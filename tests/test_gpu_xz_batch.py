"""The batched XZ decoder (swc_xz_unarchive_batch) and swc_crc64_batch against the oracle's xz_unarchive / crc64 and the
single-archive swc_xz_unarchive: status, output length and bytes unit by unit on the catalogue of tests/xz_cases.py, every
byte cut of its small archives, hostile layouts, output overflow and rerun, a CUDA-graph capture and the config-5 shape
(1 MiB archives against the raw LZMA2 batch on their block payloads)."""
import ctypes as C
import random

import numpy as np
import pytest

import helpers as H
import xz_cases as X

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


def _run(datas, caps):
    from swcompression_b200.batch import Batch
    b = Batch.from_units("xz", datas, caps)
    b.run()
    st, ln, used = b.results()
    assert (used == 0).all()
    return b, st, ln, b.outputs()


def _single(data):
    from swcompression_b200 import _lib
    buf, n = _lib.inbuf(data)
    out, ol = C.c_void_p(), C.c_size_t()
    st = _lib.lib().swc_xz_unarchive(buf, n, C.byref(out), C.byref(ol))
    return st, _lib.take(out, ol)


def _compare(expect, st, ln, outs):
    bad = []
    for i, (est, eout) in enumerate(expect):
        if st[i] != est:
            bad.append((i, "status", int(st[i]), est))
        elif ln[i] != len(eout) or outs[i] != eout:
            bad.append((i, "out_len/bytes", int(ln[i]), len(eout)))
    return bad


def test_catalogue(S, oracle):
    """the whole catalogue as one batch: the oracle's status, out_len and bytes (OK and WRONG_CHECK), the single call's status
    and bytes, SWC_ERR_UNSUPPORTED for the chains and chunks the batch does not run"""
    arcs = X.cases()
    expect = [X.expected(oracle, a) for a in arcs]
    spare = max(len(oracle.xz_unarchive(a.data)[1]) for a in arcs) + 4096      # a failing unit may decode blocks first
    caps = np.array([len(o) + 64 if s in (X.OK,) + X.PAYLOAD_CARRYING else spare for s, o in expect], dtype=np.uint64)
    _, st, ln, outs = _run([a.data for a in arcs], caps)
    bad = _compare(expect, st, ln, outs)
    assert not bad, f"{len(bad)} of {len(arcs)} differ: {[(arcs[x[0]].name,) + x[1:] for x in bad[:8]]}"
    for i, a in enumerate(arcs):
        sst, sout = _single(a.data)
        ost, oout, _ = oracle.xz_unarchive(a.data)
        assert sst == ost, a.name
        if not a.unsupported:
            assert st[i] == sst and (sst not in (X.OK,) + X.PAYLOAD_CARRYING or sout == outs[i]), a.name
        else:
            assert st[i] == X.UNSUPPORTED, a.name


def test_truncations(S, oracle):
    """every byte cut of the catalogue's archives under 4 KiB and of the archives the batch refuses, as one batch, the rest of
    the archive lying behind the unit in memory: the oracle's status (REFERENCE_TRAP included) and bytes, and for a refused
    archive SWC_ERR_UNSUPPORTED only from the cut that reaches the refused block's filter chain or chunk (every earlier error
    wins); a seeded sample also against swc_xz_unarchive"""
    units, tails, caps, expect = [], [], [], []
    for a in X.cases():
        if len(a.data) >= 4096 and not a.unsupported:
            continue
        ost, out, _ = oracle.xz_unarchive(a.data)
        cap = len(out) + 16 if ost in (X.OK,) + X.PAYLOAD_CARRYING else 16384      # a cut decodes no more than the whole
        for k in range(len(a.data) + 1):
            units.append(a.data[:k]); tails.append(a.data[k:]); caps.append(cap)
            expect.append(X.expected(oracle, a, k))
    assert sum(e[0] == X.UNSUPPORTED for e in expect) > 1000 and sum(e[0] == X.XZ_PADDING for e in expect) > 10
    from swcompression_b200.batch import Batch
    buf, offs, lens = H.pack_hostile(units, random.Random(93), None, tails)
    b = Batch("xz", buf, offs, lens, np.array(caps, dtype=np.uint64))
    b.run()
    st, ln, _ = b.results()
    outs = b.outputs()
    bad = _compare(expect, st, ln, outs)
    assert not bad, (len(units), bad[:8])
    assert (st == X.TRAP).sum() > 1000
    for i in random.Random(94).sample(range(len(units)), 1500):
        if st[i] != X.UNSUPPORTED:
            assert _single(units[i])[0] == st[i], i


def _hostile_units(rng):
    """-> (units, tails): whole, cut and bit-flipped archives of the catalogue's valid ones"""
    units, tails = [], []
    good = [a.data for a in X.cases() if a.status == X.OK and not a.unsupported and 0 < len(a.data) < 40000]
    for j in range(120):
        a = good[j % len(good)]
        if j % 4 == 1:
            c = rng.randrange(1, len(a))
            units.append(a[:c]); tails.append(a[c:])
        elif j % 4 == 2:
            b = bytearray(a); b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            units.append(bytes(b)); tails.append(None)
        else:
            units.append(a); tails.append(b"\xFD7zXZ\x00" if j % 2 else None)
    return units, tails


def _hostile_run(units, tails, expect, rng, aligned, spare):
    import torch
    from swcompression_b200 import _lib
    sizes = [len(o) if s in (X.OK,) + X.PAYLOAD_CARRYING else None for s, o in expect]
    out_off, out_cap, total = H.fenced_layout(sizes, spare)
    if aligned:
        buf, offs, lens = H.pack_hostile(units, rng, None, tails, residues=[0] * len(units))
    else:
        buf, offs, lens = H.pack_hostile(units, rng, None, tails)
    n = len(units)
    d_in, d_off, d_len, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_ln = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    assert _lib.lib().swc_xz_unarchive_batch(_p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_oo), _p(d_oc), _p(d_ln), _p(d_st),
                                             n, _stream()) == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    st, ln = d_st.cpu().numpy(), d_ln.cpu().numpy()
    outs = [bytes(out[int(o):int(o) + int(c)]) for o, c in zip(out_off, out_cap)]
    return st, ln, outs, out_cap, H.fence_violations(out, out_off, out_cap)


def test_hostile_layout(S, oracle):
    """units at every start residue and back to back, cut archives followed by their own rest, damaged archives, output
    capacities exact, 1-15 short (overflow with the declared size) and 1-15 long, between sentinel bytes that must stay
    intact; the same units packed 16-byte aligned give the same results"""
    rng = random.Random(95)
    units, tails = _hostile_units(rng)
    expect = [X.expected(oracle, X.Arc("h", u)) for u in units]
    # a damaged unit may decode all its blocks before it fails (a damaged index): room for the whole original
    spare = max(len(oracle.xz_unarchive(a.data)[1]) for a in X.cases() if a.status == X.OK and 0 < len(a.data) < 40000) + 1024
    st, ln, outs, caps, fence = _hostile_run(units, tails, expect, rng, False, spare)
    bad = []
    for i, (est, eout) in enumerate(expect):
        if est in (X.OK,) + X.PAYLOAD_CARRYING and len(eout) > caps[i]:
            if st[i] != X.OVERFLOW or (est == X.OK and ln[i] != len(eout)):
                bad.append((i, "overflow", int(st[i]), int(ln[i]), len(eout)))
        elif st[i] != est or ln[i] != len(eout) or outs[i][:len(eout)] != eout:
            bad.append((i, int(st[i]), est, int(ln[i]), len(eout)))
    assert not bad and fence.size == 0, (bad[:8], fence[:8])
    assert (st == X.OVERFLOW).sum() > 5
    st2, ln2, outs2, _, fence2 = _hostile_run(units, tails, expect, random.Random(95), True, spare)
    assert (st2 == st).all() and (ln2 == ln).all() and fence2.size == 0
    assert all(a[:int(n)] == b[:int(n)] for a, b, n, s in zip(outs, outs2, ln, st) if s != X.OVERFLOW)


def test_output_overflow_then_rerun(S, oracle):
    """valid archives (multi-stream ones too) given size - 1 report SWC_ERR_OUTPUT_OVERFLOW with out_len = the declared size;
    a rerun at that size decodes; an archive whose index is damaged reports the overflow with out_len 0"""
    arcs = [a for a in X.cases() if a.status == X.OK and not a.unsupported and len(oracle.xz_unarchive(a.data)[1]) > 0]
    assert sum(a.name.startswith("three streams") for a in arcs) == 3
    datas = [a.data for a in arcs]
    sizes = [len(oracle.xz_unarchive(d)[1]) for d in datas]
    _, st, ln, _ = _run(datas, np.array([s - 1 for s in sizes], dtype=np.uint64))
    assert (st == X.OVERFLOW).all() and list(ln) == sizes
    _, st, ln, outs = _run(datas, ln.astype(np.uint64))
    assert (st == 0).all() and outs == [oracle.xz_unarchive(d)[1] for d in datas]
    from test_framing_handmade import GOOD, RAW
    damaged = bytearray(GOOD)
    damaged[-12 - 10] ^= 0x10                                       # the index record's Unpadded Size: the backward walk misses
    _, st, ln, _ = _run([bytes(damaged)], np.array([len(RAW) - 1], dtype=np.uint64))
    assert st[0] == X.OVERFLOW and ln[0] == 0


def test_graph_capture(S, oracle):
    """the call is one enqueue with no host synchronisation or allocation: captured into a CUDA graph, the replay gives the
    eager results"""
    import torch
    arcs = [a for a in X.cases() if not a.unsupported][:150]
    datas = [a.data for a in arcs]
    spare = max(len(oracle.xz_unarchive(d)[1]) for d in datas) + 4096                # no unit overflows
    from swcompression_b200.batch import Batch
    b = Batch.from_units("xz", datas, spare)
    b.run()
    st0, ln0, _ = b.results()
    outs0 = b.outputs()
    assert not _compare([X.expected(oracle, a) for a in arcs], st0, ln0, outs0)
    b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_out.zero_()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b.run()
    torch.cuda.synchronize()
    assert (b.d_status.cpu().numpy() == -1).all()
    g.replay()
    st1, ln1, _ = b.results()
    assert (st1 == st0).all() and (ln1 == ln0).all() and b.outputs() == outs0


def test_crc64_batch(S, oracle):
    """swc_crc64_batch equals the oracle's CRC-64 for lengths 0-300 and around the 32 x 16-byte segment multiples, at every
    start residue; units whose status is not 0 are skipped and left at 0"""
    import torch
    from swcompression_b200 import _lib
    rng = random.Random(96)
    lens = list(range(301)) + [m * 512 + d for m in (1, 2, 3, 64) for d in (-17, -1, 0, 1, 16)] + [(1 << 20) + 3]
    units = [H.random_bytes(rng, n) if n < 40000 else np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
             for n in lens]
    buf, offs, ulens = H.pack_hostile(units, rng)
    n = len(units)
    status = np.zeros(n, dtype=np.int32)
    status[5::13] = 807
    d_buf, d_off, d_len, d_st = _dev(buf), _dev(offs), _dev(ulens), _dev(status)
    d_res = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    L = _lib.lib()
    assert L.swc_crc64_batch(_p(d_buf), _p(d_off), _p(d_len), _p(d_st), _p(d_res), n, _stream()) == 0
    assert L.swc_crc64_batch(_p(d_buf), _p(d_off), _p(d_len), None, None, n, _stream()) == 4
    torch.cuda.synchronize()
    got = d_res.cpu().numpy().view(np.uint64)
    want = [0 if status[i] else oracle.crc64(u) for i, u in enumerate(units)]
    bad = [(i, len(units[i])) for i in range(n) if int(got[i]) != want[i]]
    assert not bad, bad[:8]


def _config5(count):
    """`count` archives of 1 MiB (CRC-64, preset 6, 1 MiB dictionary), from 16 distinct inputs -> (archives, raw inputs)"""
    import lzma
    raws = [H.textlike(1 << 20, 970 + k) for k in range(16)]
    arcs = [lzma.compress(r, format=lzma.FORMAT_XZ, check=lzma.CHECK_CRC64,
                          filters=[{"id": lzma.FILTER_LZMA2, "preset": 6, "dict_size": 1 << 20}]) for r in raws]
    return [arcs[i % 16] for i in range(count)], [raws[i % 16] for i in range(count)]


def block_payload(arc):
    """the single block's LZMA2 payload and dictionary byte of a one-block archive from Python's lzma"""
    hsz = (arc[12] + 1) * 4
    hdr = arc[12:12 + hsz]
    k = hdr.index(b"\x21\x01", 2)
    return arc[12 + hsz:], hdr[k + 2]


def test_config5_shape(S, oracle):
    """1 184 archives of 1 MiB give the bytes swc_lzma2_decompress_batch gives on their block payloads; a seeded sample equals
    the oracle"""
    from swcompression_b200.batch import Batch
    arcs, raws = _config5(1184)
    b, st, ln, _ = _run(arcs, 1 << 20)
    assert (st == 0).all() and (ln == 1 << 20).all()
    payloads = [block_payload(a) for a in arcs[:16]]
    r = Batch.from_units("lzma2", [p for p, _ in payloads], 1 << 20, aux=bytes(d for _, d in payloads))
    r.run()
    rst, rln, _ = r.results()
    assert (rst == 0).all()
    xo = b.d_out.view(-1)[: 1184 << 20].view(1184, 1 << 20)
    ro = r.d_out.view(-1)[: 16 << 20].view(16, 1 << 20)
    import torch
    assert torch.equal(xo, ro.repeat(74, 1))
    for i in random.Random(97).sample(range(1184), 3):
        assert bytes(xo[i].cpu().numpy()) == oracle.xz_unarchive(arcs[i])[1] == raws[i]
