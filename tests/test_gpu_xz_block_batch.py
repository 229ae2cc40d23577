"""The block-parallel XZ batch (swc_xz_block_unarchive_batch, Batch codec 'xz_blocks') against the oracle and against
swc_xz_unarchive_batch ('xz') on the same bytes and capacities: status, out_len and bytes unit by unit, and parallel_blocks,
which must show that every valid unit with room in the block table went through the block stage.  Covers the catalogues of
tests/xz_cases.py and tests/xz_block_cases.py, every byte cut of their archives under 4 KiB with the rest of the archive
behind the unit, output overflow and rerun, the block table's capacity, caller and library scratch, hostile layouts with
fenced outputs, a CUDA-graph replay, an archive whose output passes 4 GiB, and a .tar.xz walked in place by Batch.tar_of."""
import ctypes as C
import io
import random
import tarfile
import zlib

import numpy as np
import pytest

import helpers as H
import xz_block_cases as XB
import xz_cases as X

pytestmark = pytest.mark.gpu
CARRY = (X.OK,) + X.PAYLOAD_CARRYING
INVALID_ARG = 4


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


def _both(buf, offs, lens, caps, max_blocks=None):
    """-> ('xz' results, 'xz_blocks' results, parallel_blocks, the 'xz_blocks' batch); results = (status, out_len, outputs)"""
    from swcompression_b200.batch import Batch
    res = []
    for codec in ("xz", "xz_blocks"):
        b = Batch(codec, buf, offs, lens, np.asarray(caps, dtype=np.uint64), max_blocks=max_blocks if codec == "xz_blocks" else None)
        b.run()
        st, ln, _ = b.results()
        host = b.d_out.cpu().numpy()
        outs = [bytes(host[int(o):int(o) + min(int(l), int(c))]) for o, l, c in zip(b.h_out_off, ln, b.h_out_cap)]
        res.append((st, ln, outs))
    return res[0], res[1], b.parallel_blocks(), b


def _units(units, caps, max_blocks=None):
    from swcompression_b200.batch import pack_units
    buf, offs, lens = pack_units(units)
    return _both(buf, offs, lens, caps, max_blocks)


def _same(old, new):
    """unit indices where the two batches differ in status, out_len or the bytes [0, out_len) on OK / WRONG_CHECK"""
    return [i for i in range(len(old[0])) if old[0][i] != new[0][i] or old[1][i] != new[1][i]
            or (old[0][i] in CARRY and old[2][i] != new[2][i])]


def _blocks(data):
    w = XB.back_walk(data)
    return 0 if w is None else len(w)


def _qualifies(data, cap):
    w = XB.back_walk(data)
    return w is not None and sum(n for _, n, _ in w) <= cap


def _expected_parallel(units, caps, st, max_blocks=None):
    """the place rule restated: qualifying units take table entries in unit order; a unit is placed iff its records end
    inside the table; a placed unit that comes out SWC_OK took the block path"""
    at, out = 0, []
    for u, c, s in zip(units, caps, st):
        q = _qualifies(u, int(c))
        nb = _blocks(u) if q else 0
        placed = q and (max_blocks is None or at + nb <= max_blocks)
        out.append(nb if placed and s == X.OK else 0)
        at += nb
    return np.array(out, dtype=np.uint32)


def _caps_for(oracle, arcs):
    expect = [X.expected(oracle, a) for a in arcs]
    spare = max(len(oracle.xz_unarchive(a.data)[1]) for a in arcs) + 4096
    return expect, np.array([len(o) + 64 if s in CARRY else spare for s, o in expect], dtype=np.uint64)


def test_catalogue(S, oracle):
    """both catalogues as one batch: the oracle's answers, 'xz''s answers, and parallel_blocks = the block count of every
    valid unit (one of them a stream of zero blocks, others of 64)"""
    arcs = X.cases() + XB.cases()
    expect, caps = _caps_for(oracle, arcs)
    old, new, par, _ = _units([a.data for a in arcs], caps)
    assert not _same(old, new), [arcs[i].name for i in _same(old, new)[:8]]
    bad = [(a.name, int(new[0][i]), e[0]) for i, (a, e) in enumerate(zip(arcs, expect))
           if new[0][i] != e[0] or (e[0] in CARRY and new[2][i] != e[1])]
    assert not bad, bad[:8]
    want = _expected_parallel([a.data for a in arcs], caps, new[0])
    assert (par == want).all(), [(arcs[i].name, int(par[i]), int(want[i])) for i in np.nonzero(par != want)[0][:8]]
    assert (par >= 64).sum() >= 3 and (par > 1).sum() > 40


def test_truncations(S, oracle):
    """every byte cut of both catalogues' archives under 4 KiB, the rest of the archive lying behind the unit: a cut unit
    never validates from bytes outside it"""
    units, tails, caps, expect = [], [], [], []
    for a in X.cases() + XB.cases():
        if len(a.data) >= 4096 and not a.unsupported:
            continue
        ost, out, _ = oracle.xz_unarchive(a.data)
        cap = len(out) + 16 if ost in CARRY else 16384
        for k in range(len(a.data) + 1):
            units.append(a.data[:k]); tails.append(a.data[k:]); caps.append(cap)
            expect.append(X.expected(oracle, a, k))
    buf, offs, lens = H.pack_hostile(units, random.Random(130), None, tails)
    old, new, par, _ = _both(buf, offs, lens, caps)
    assert not _same(old, new), _same(old, new)[:8]
    bad = [i for i, e in enumerate(expect) if new[0][i] != e[0] or (e[0] in CARRY and new[2][i] != e[1])]
    assert not bad, bad[:8]
    want = _expected_parallel(units, caps, new[0])
    assert (par == want).all(), np.nonzero(par != want)[0][:8]
    assert (par > 0).sum() > 50


def test_overflow_then_rerun(S, oracle):
    """valid multi-block archives at every capacity below their size (small outputs), or at 0, 1, each block boundary +-1
    and size - 1: the old batch's status and out_len (the declared size); a rerun at out_len decodes block-parallel"""
    arcs = [a for a in XB.cases() + X.cases() if a.status == X.OK and not a.unsupported and _blocks(a.data) > 0
            and len(oracle.xz_unarchive(a.data)[1]) > 0][:40]
    units, caps = [], []
    for a in arcs:
        size = len(oracle.xz_unarchive(a.data)[1])
        if size <= 4096:
            cs = range(size)
        else:
            marks = {0, 1, size - 1}
            for _, _, at in XB.back_walk(a.data):
                marks |= {at - 1, at, at + 1}
            cs = sorted(c for c in marks if 0 <= c < size)
        for c in cs:
            units.append(a.data); caps.append(c)
    old, new, par, _ = _units(units, caps)
    assert not _same(old, new)
    assert (new[0] == X.OVERFLOW).all() and (par == 0).all()
    assert [int(x) for x in new[1]] == [len(oracle.xz_unarchive(u)[1]) for u in units]
    datas = [a.data for a in arcs]
    old, new, par, _ = _units(datas, [len(oracle.xz_unarchive(d)[1]) for d in datas])
    assert (new[0] == 0).all() and new[2] == [oracle.xz_unarchive(d)[1] for d in datas]
    assert [int(p) for p in par] == [_blocks(d) for d in datas]


def test_max_blocks(S, oracle):
    """the table's capacity changes the path, never the results: library-counted (0), exact, exact - 1 (the last unit falls
    back), 1; a caller scratch one byte short is refused; no scratch takes the pool"""
    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import pack_units
    arcs = [a for a in XB.cases() if a.status == X.OK and _blocks(a.data) > 1][:12]
    datas = [a.data for a in arcs] + [arcs[0].data]
    total = sum(_blocks(d) for d in datas)
    caps = np.array([len(oracle.xz_unarchive(d)[1]) + 32 for d in datas], dtype=np.uint64)
    ref = None
    for mb in (None, total, total - 1, 1):
        old, new, par, _ = _units(datas, caps, mb)
        assert not _same(old, new) and (new[0] == 0).all(), mb
        want = _expected_parallel(datas, caps, new[0], mb)
        assert (par == want).all(), (mb, par, want)
        if mb == total - 1:
            assert par[-1] == 0 and (par[:-1] > 0).all()
        if ref is None:
            ref = new
        assert new[2] == ref[2]
    buf, offs, lens = pack_units(datas)
    n = len(datas)
    L = _lib.lib()
    d_in, d_off, d_len = _dev(buf), _dev(offs), _dev(lens)
    out_off = np.concatenate([[0], np.cumsum(caps[:-1])]).astype(np.uint64)
    d_oo, d_oc = _dev(out_off), _dev(caps)
    d_out = torch.zeros(int(caps.sum()) + 64, dtype=torch.uint8, device="cuda")
    d_ln = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_par = torch.zeros(n, dtype=torch.int32, device="cuda")
    need = L.swc_xz_block_batch_scratch_bytes(n, total)
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    args = lambda: (_p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_oo), _p(d_oc), _p(d_ln), _p(d_st), _p(d_par), n, total)
    assert L.swc_xz_block_unarchive_batch(*args(), _p(scr), need - 1, _stream()) == INVALID_ARG
    assert L.swc_xz_block_unarchive_batch(*args(), None, 0, _stream()) == 0
    torch.cuda.synchronize()
    assert (d_st.cpu().numpy() == 0).all() and [int(p) for p in d_par.cpu().numpy()] == [_blocks(d) for d in datas]
    d_st.fill_(-1); d_par.zero_()
    assert L.swc_xz_block_unarchive_batch(*args(), _p(scr), need, _stream()) == 0
    torch.cuda.synchronize()
    assert (d_st.cpu().numpy() == 0).all() and [int(p) for p in d_par.cpu().numpy()] == [_blocks(d) for d in datas]
    out = d_out.cpu().numpy()
    assert [bytes(out[int(o):int(o) + len(r)]) for o, r in zip(out_off, ref[2])] == ref[2]


def _hostile_units(rng):
    units, tails = [], []
    good = [a.data for a in XB.cases() + X.cases() if a.status == X.OK and not a.unsupported and 0 < len(a.data) < 40000]
    for j in range(160):
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


def test_hostile_layout(S, oracle):
    """units at every start residue and back to back, cut archives followed by their own rest, damaged archives, output
    regions exact, 1-15 bytes short and 1-15 long between sentinel bytes: both batches give the same answers, the oracle's,
    and neither writes a byte outside a region"""
    import torch
    from swcompression_b200 import _lib
    rng = random.Random(131)
    units, tails = _hostile_units(rng)
    expect = [X.expected(oracle, X.Arc("h", u)) for u in units]
    spare = max(len(oracle.xz_unarchive(u)[1]) for u in units) + 1024
    out_off, out_cap, total = H.fenced_layout([len(o) if s in CARRY else None for s, o in expect], spare)
    buf, offs, lens = H.pack_hostile(units, rng, None, tails)
    n = len(units)
    d_in, d_off, d_len, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
    L = _lib.lib()
    res = []
    for new in (False, True):
        d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
        d_ln = torch.zeros(n, dtype=torch.int64, device="cuda")
        d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        d_par = torch.zeros(n, dtype=torch.int32, device="cuda")
        io = (_p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_oo), _p(d_oc), _p(d_ln), _p(d_st))
        if new:
            assert L.swc_xz_block_unarchive_batch(*io, _p(d_par), n, 0, None, 0, _stream()) == 0
        else:
            assert L.swc_xz_unarchive_batch(*io, n, _stream()) == 0
        torch.cuda.synchronize()
        out = d_out.cpu().numpy()
        st, ln = d_st.cpu().numpy(), d_ln.cpu().numpy()
        outs = [bytes(out[int(o):int(o) + min(int(l), int(c))]) for o, l, c in zip(out_off, ln, out_cap)]
        assert H.fence_violations(out, out_off, out_cap).size == 0, new
        res.append((st, ln, outs, d_par.cpu().numpy()))
    assert not _same(res[0][:3], res[1][:3]), _same(res[0][:3], res[1][:3])[:8]
    st, ln, outs, par = res[1]
    for i, (est, eout) in enumerate(expect):
        if est in CARRY and len(eout) > out_cap[i]:
            assert st[i] == X.OVERFLOW, i
        else:
            assert st[i] == est and (est not in CARRY or outs[i] == eout), i
    want = _expected_parallel(units, out_cap, st)
    assert (par == want).all() and (par > 0).sum() > 20


def test_graph_capture(S, oracle):
    """with a caller scratch and max_blocks > 0 the call captures into a CUDA graph; the replay gives the eager results"""
    import torch
    from swcompression_b200.batch import Batch
    arcs = [a for a in XB.cases() + X.cases() if not a.unsupported][:150]
    datas = [a.data for a in arcs]
    expect, caps = _caps_for(oracle, arcs)
    b = Batch.from_units("xz_blocks", datas, caps, max_blocks=sum(_blocks(d) for d in datas) + 7)
    assert b.d_scratch is not None
    b.run()
    st0, ln0, _ = b.results()
    outs0, par0 = b.outputs(), b.parallel_blocks().copy()
    assert all(s == e[0] and (s not in CARRY or o == e[1]) for s, o, e in zip(st0, outs0, expect))
    assert (par0 > 0).sum() > 40
    b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_out.zero_(); b.d_parallel.fill_(-1)
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
    assert (st1 == st0).all() and (ln1 == ln0).all() and b.outputs() == outs0 and (b.parallel_blocks() == par0).all()


def test_output_past_4gib(S):
    """65 blocks of 64 MiB of a repeating pattern: out_len, parallel_blocks and the output's CRC-32 (64-bit output offsets)"""
    import torch
    from swcompression_b200.batch import Batch
    mib64 = 64 << 20
    raw = (bytes(range(251)) * (mib64 // 251 + 1))[:mib64]
    payload = X.lzma2_raw(raw, preset=0, dict_size=1 << 20)
    arc = XB.stream([(payload, 0x10, raw)] * 65, X.CHECK_CRC32)
    want_crc = 0
    for _ in range(65):
        want_crc = zlib.crc32(raw, want_crc)
    b = Batch.from_units("xz_blocks", [arc], 65 * mib64)
    b.run()
    st, ln, _ = b.results()
    assert int(st[0]) == 0 and int(ln[0]) == 65 * mib64 > 1 << 32
    assert int(b.parallel_blocks()[0]) == 65
    out = b.d_out[:65 * mib64]
    assert zlib.crc32(memoryview(out.cpu().numpy())) == want_crc
    ref = torch.from_numpy(np.frombuffer(raw, dtype=np.uint8).copy()).cuda()
    assert bool((out.view(65, mib64) == ref).all())


def test_tar_xz_walked_in_place(S):
    """a .tar.xz in the shape multi-threaded xz writes (the tar cut into 3 independent blocks), decoded by 'xz_blocks' and
    walked by Batch.tar_of: the records of the plain archive through 'tar'"""
    from swcompression_b200.batch import Batch
    rng = random.Random(132)
    bio = io.BytesIO()
    with tarfile.open(fileobj=bio, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for k in range(7):
            data = H.textlike(rng.randrange(0, 40000), 133 + k)
            ti = tarfile.TarInfo(f"dir/file{k}.txt")
            ti.size, ti.mtime = len(data), 1700000000 + k
            tf.addfile(ti, io.BytesIO(data))
    plain = bio.getvalue()
    third = len(plain) // 3
    parts = [plain[:third], plain[third:2 * third], plain[2 * third:]]
    arc = XB.stream([(X.lzma2_raw(p), 0x10, p) for p in parts], X.CHECK_CRC64, sizes=[True] * 3)
    x = Batch.from_units("xz_blocks", [arc, arc], len(plain) + 512)
    t = Batch.tar_of(x)
    x.run()
    t.run()
    st, ln, _ = x.results()
    assert (st == 0).all() and (ln == len(plain)).all() and list(x.parallel_blocks()) == [3, 3]
    p = Batch.from_units("tar", [plain], None)
    p.run()
    assert [int(v[0]) for v in p.tar_results()] == [int(v[0]) for v in t.tar_results()]
    assert int(t.tar_results()[0][0]) >= 7 and t.records(0) == t.records(1) == p.records(0)
