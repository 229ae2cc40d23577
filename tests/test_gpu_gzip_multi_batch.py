"""The member-parallel gzip batch (swc_gzip_multi_unarchive_batch, Batch codec 'gzip_multi') against the oracle's
multiUnarchive walk: status, output bytes, out_len, consumed bytes and the member table unit by unit, and parallel_members,
which must equal the member count of every BGZF file and clean concatenation and fall short where a look-alike sits outside
BGZF.  Covers the catalogue of tests/gzip_member_cases.py, every byte cut of its files under 4 KiB with the rest of the file
behind the unit, a member table too small for the batch, caller scratch against the library pool, overflow and rerun,
hostile layouts with fenced outputs, a CUDA-graph replay, a file whose output passes 4 GiB, and a BGZF .tar.gz walked in place
by Batch.tar_of."""
import ctypes as C
import io
import random
import tarfile
import zlib

import numpy as np
import pytest

import gzip_member_cases as G
import helpers as H

pytestmark = pytest.mark.gpu
CARRY = (G.OK, G.GZ_CRC)
OVERFLOW = 1


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


def _caps(expect, datas, most=1 << 22):
    """room for the output on OK / wrongCRC, and for everything the walk may write before an error otherwise"""
    return np.array([len(e[1]) + 16 if e[0] in CARRY else min(len(d) * 1032 + 64, most) for e, d in zip(expect, datas)],
                    dtype=np.uint64)


def _no_tiny(ends):
    """no member decodes to 1-15 bytes (such a member and those behind it take the sequential walk)"""
    sizes = [b - a for a, b in zip([0] + ends[:-1], ends)]
    return all(x == 0 or x >= 16 for x in sizes)


def _run(units, caps, **kw):
    """-> (status, out_len, consumed, outputs, tables, parallel_members, batch) of a 'gzip_multi' batch"""
    from swcompression_b200.batch import Batch
    b = Batch.from_units("gzip_multi", units, caps, **kw)
    b.run()
    st, ln, used = b.results()
    host = b.d_out.cpu().numpy()
    outs = [bytes(host[int(o):int(o) + min(int(l), int(c))]) for o, l, c in zip(b.h_out_off, ln, b.h_out_cap)]
    return st, ln, used, outs, [b.member_table(i) for i in range(b.n)], b.parallel_members().copy(), b


def _mismatches(res, expect, names):
    st, ln, used, outs, tables = res[:5]
    bad = []
    for i, e in enumerate(expect):
        est, eout, ends, starts, consumed = e
        got = (int(st[i]), int(used[i]), tables[i] if est in CARRY else None, outs[i] if est in CARRY else None,
               int(ln[i]) if est in CARRY else 0)
        want = (est, consumed, (ends, starts) if est in CARRY else None, eout if est in CARRY else None,
                len(eout) if est in CARRY else 0)
        if est not in CARRY:
            got = got[:2] + (None, None, int(ln[i]))
        if got != want:
            bad.append((names[i], got[:2], want[:2]))
    return bad


def test_catalogue(S, oracle):
    """the whole catalogue as one batch: the oracle's answers; parallel_members = the member count of every BGZF file and
    clean concatenation, and less for the plain files with planted look-alikes"""
    cases = G.cases()
    expect = [G.expect(oracle, c.data) for c in cases]
    res = _run([c.data for c in cases], _caps(expect, [c.data for c in cases]))
    bad = _mismatches(res, expect, [c.name for c in cases])
    assert not bad, bad[:8]
    par = res[5]
    for i, (c, e) in enumerate(zip(cases, expect)):
        if e[0] == G.OK and _no_tiny(e[2]) and (c.name.startswith("bgzf") or c.name.startswith("concatenation") or "fname" in c.name):
            assert par[i] == len(e[2]), (c.name, int(par[i]), len(e[2]))
        if e[0] == G.OK and (c.name.startswith("plain look-alikes") or c.name.startswith("look-alike in member 0")):
            assert par[i] < len(e[2]), c.name


def test_truncations(S, oracle):
    """every byte cut of the catalogue's files under 4 KiB, the rest of the file lying behind the unit"""
    cuts = G.cuts()
    full = {c.name: c.data for c in G.cases()}
    units = [d for _, d in cuts]
    tails = [full[name.rsplit(" cut ", 1)[0]][len(d):] for name, d in cuts]
    expect = [G.expect(oracle, d) for d in units]
    from swcompression_b200.batch import Batch
    buf, offs, lens = H.pack_hostile(units, random.Random(140), None, tails)
    # a cut never writes more than its whole file decodes to: the room of the whole file's output suffices
    whole = {name: len(G.expect(oracle, data)[1]) for name, data in full.items()}
    caps = np.array([whole[name.rsplit(" cut ", 1)[0]] + 16 for name, _ in cuts], dtype=np.uint64)
    b = Batch("gzip_multi", buf, offs, lens, np.maximum(caps, _caps(expect, units, 1 << 16)))
    b.run()
    st, ln, used = b.results()
    host = b.d_out.cpu().numpy()
    outs = [bytes(host[int(o):int(o) + min(int(l), int(c))]) for o, l, c in zip(b.h_out_off, ln, b.h_out_cap)]
    res = (st, ln, used, outs, [b.member_table(i) for i in range(b.n)])
    bad = _mismatches(res, expect, [n for n, _ in cuts])
    assert not bad, bad[:8]


def test_max_members(S, oracle):
    """a candidate table too small for the batch (1, half) and the library's count give the same results"""
    cases = G.cases()
    datas = [c.data for c in cases]
    expect = [G.expect(oracle, d) for d in datas]
    caps = _caps(expect, datas)
    base = _run(datas, caps)
    assert not _mismatches(base, expect, [c.name for c in cases])
    total = sum(len(G.zlib_starts(d) or [0]) for d in datas)
    for mm in (1, total // 2, 10 * total):
        res = _run(datas, caps, max_members=mm)
        assert not _mismatches(res, expect, [c.name for c in cases]), mm
        if mm == 1:
            assert (res[5] <= 1).all()


def test_caller_scratch_and_pool(S, oracle):
    """a caller scratch with max_members = 0 (the library counts, the table the largest that fits), a caller scratch with a
    fixed table, and the pool: the same results; a caller scratch smaller than the tables is refused"""
    from swcompression_b200 import _lib
    from swcompression_b200.batch import Batch
    cases = G.cases()
    datas = [c.data for c in cases]
    expect = [G.expect(oracle, d) for d in datas]
    caps = _caps(expect, datas)
    pool = _run(datas, caps)
    b = Batch.from_units("gzip_multi", datas, caps)
    need = _lib.lib().swc_gzip_member_batch_scratch_bytes(b.n, 4096, b.out_total)
    for kw in (dict(scratch_bytes=need), dict(max_members=4096), dict(max_members=4096, scratch_bytes=need)):
        res = _run(datas, caps, **kw)
        assert all((x == y).all() if isinstance(x, np.ndarray) else x == y for x, y in zip(res[:6], pool[:6])), kw
    tiny = Batch.from_units("gzip_multi", datas, caps, max_members=64, scratch_bytes=256)
    with pytest.raises(RuntimeError):
        tiny.run()


def test_overflow_then_rerun(S, oracle):
    """valid files at capacities below their size: SWC_ERR_OUTPUT_OVERFLOW with out_len the exact size; a rerun at out_len
    is final and exact"""
    cases = [c for c in G.cases() if c.status in (G.OK, G.GZ_CRC) and 0 < len(G.expect(oracle, c.data)[1]) < 400000][:30]
    units, caps, expect = [], [], []
    for c in cases:
        e = G.expect(oracle, c.data)
        size = len(e[1])
        for cap in sorted({0, 1, size // 3, size // 2, size - 1}):
            if cap < size:
                units.append(c.data); caps.append(cap); expect.append(e)
    res = _run(units, np.array(caps, dtype=np.uint64))
    st, ln = res[0], res[1]
    assert (st == OVERFLOW).all(), st
    for i, e in enumerate(expect):
        if e[0] == G.OK:
            assert int(ln[i]) == len(e[1]), i
        else:
            assert int(ln[i]) >= len(e[1]), i
    res = _run(units, np.asarray(ln, dtype=np.uint64))
    assert not _mismatches(res, expect, [str(i) for i in range(len(units))])


def test_hostile_layout(S, oracle):
    """units at every start residue and back to back, cut files followed by their own rest, output regions exact, 1-15 bytes
    short and 1-15 long between sentinel bytes: the oracle's answers (overflow where the region is short), and no byte
    written outside a region"""
    import torch
    from swcompression_b200 import _lib
    rng = random.Random(141)
    units, tails = [], []
    for c in G.cases():
        if len(c.data) > 60000:
            continue
        k = rng.randrange(len(c.data) + 1) if c.data and rng.random() < 0.3 else len(c.data)
        units.append(c.data[:k]); tails.append(c.data[k:] or None)
    expect = [G.expect(oracle, u) for u in units]
    out_off, out_cap, total = H.fenced_layout([len(e[1]) if e[0] in CARRY else None for e in expect], 1 << 20)
    buf, offs, lens = H.pack_hostile(units, rng, None, tails)
    n = len(units)
    mcap = np.asarray(lens, dtype=np.uint64) // np.uint64(20) + np.uint64(1)
    moff = np.concatenate([[0], np.cumsum(mcap[:-1])]).astype(np.uint64)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_ln, d_used, d_nm = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(3))
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    d_end, d_start = (torch.zeros(int(mcap.sum()), dtype=torch.int64, device="cuda") for _ in range(2))
    d_par = torch.zeros(n, dtype=torch.int32, device="cuda")
    keep = [_dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap), _dev(moff), _dev(mcap)]
    d_in, d_off, d_len, d_oo, d_oc, d_moff, d_mcap = keep
    st = _lib.lib().swc_gzip_multi_unarchive_batch(
        _p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_oo), _p(d_oc), _p(d_ln), _p(d_used), _p(d_st), _p(d_nm), _p(d_moff),
        _p(d_mcap), _p(d_end), _p(d_start), _p(d_par), n, 0, None, 0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    assert H.fence_violations(out, out_off, out_cap).size == 0
    sts, lns, used = d_st.cpu().numpy(), d_ln.cpu().numpy(), d_used.cpu().numpy()
    for i, e in enumerate(expect):
        if e[0] in CARRY and len(e[1]) > out_cap[i]:
            assert sts[i] == OVERFLOW and int(lns[i]) >= len(e[1]), i
        else:
            got = bytes(out[int(out_off[i]):int(out_off[i]) + int(lns[i])]) if sts[i] in CARRY else b""
            assert (int(sts[i]), int(used[i]), got) == (e[0], e[4], e[1]), i


def test_graph_capture(S, oracle):
    """with a caller scratch and max_members > 0 the call captures into a CUDA graph; the replay gives the eager results"""
    import torch
    from swcompression_b200.batch import Batch
    cases = G.cases()
    datas = [c.data for c in cases]
    expect = [G.expect(oracle, d) for d in datas]
    b = Batch.from_units("gzip_multi", datas, _caps(expect, datas), max_members=20000)
    b.run()
    st0, ln0, used0 = b.results()
    outs0, par0 = b.outputs(), b.parallel_members().copy()
    assert all(s == e[0] for s, e in zip(st0, expect))
    b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_out.zero_(); b.d_parallel.fill_(-1); b.d_consumed.zero_()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b.run()
    torch.cuda.synchronize()
    assert (b.d_status.cpu().numpy() == -1).all()
    g.replay()
    st1, ln1, used1 = b.results()
    assert (st1 == st0).all() and (ln1 == ln0).all() and (used1 == used0).all()
    assert b.outputs() == outs0 and (b.parallel_members() == par0).all()


def test_output_past_4gib(S):
    """65 members of 64 MiB of zeros in one file: out_len, parallel_members, the member table and the output's CRC-32"""
    import torch
    from swcompression_b200.batch import Batch
    import unarchive_cases as U
    mib64 = 64 << 20
    member = U.gzip_member(bytes(mib64), level=1)
    b = Batch.from_units("gzip_multi", [member * 65], 65 * mib64)
    b.run()
    st, ln, used = b.results()
    assert int(st[0]) == 0 and int(ln[0]) == 65 * mib64 > 1 << 32 and int(used[0]) == 65 * len(member)
    assert int(b.parallel_members()[0]) == 65
    ends, starts = b.member_table(0)
    assert ends == [(k + 1) * mib64 for k in range(65)] and starts == [k * len(member) for k in range(65)]
    out = b.d_out[:65 * mib64]
    assert not bool(out.any())
    assert zlib.crc32(memoryview(out[-mib64:].cpu().numpy())) == zlib.crc32(bytes(mib64))


def test_bgzf_tar_gz_walked_in_place(S):
    """a BGZF .tar.gz decoded by 'gzip_multi' and walked by Batch.tar_of: the records of the plain archive through 'tar',
    and members(i) as GzipArchive.multiUnarchive returns them"""
    from swcompression_b200.api import GzipArchive
    from swcompression_b200.batch import Batch
    rng = random.Random(142)
    bio = io.BytesIO()
    with tarfile.open(fileobj=bio, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for k in range(7):
            data = H.textlike(rng.randrange(0, 90000), 143 + k)
            ti = tarfile.TarInfo(f"dir/file{k}.txt")
            ti.size, ti.mtime = len(data), 1700000000 + k
            tf.addfile(ti, io.BytesIO(data))
    plain = bio.getvalue()
    arc, parts = G.bgzf(plain)
    x = Batch.from_units("gzip_multi", [arc, arc], len(plain) + 512, max_members=1024)
    t = Batch.tar_of(x)
    x.run()
    t.run()
    st, ln, _ = x.results()
    assert (st == 0).all() and (ln == len(plain)).all() and list(x.parallel_members()) == [len(parts)] * 2
    p = Batch.from_units("tar", [plain], None)
    p.run()
    assert [int(v[0]) for v in p.tar_results()] == [int(v[0]) for v in t.tar_results()]
    assert int(t.tar_results()[0][0]) >= 7 and t.records(0) == t.records(1) == p.records(0)
    want = GzipArchive.multiUnarchive(arc)
    got = x.members(0)
    assert [m.data for m in got] == [m.data for m in want] == parts
    assert [vars(m.header) for m in got] == [vars(m.header) for m in want]


def test_small_regions_next_to_a_neighbour(S, oracle):
    """units packed back to back, each followed directly by the next one's region: the first unit's out_cap ends 1, 2 or 5
    bytes into a member (or one member decodes to 1, 2 or 5 bytes), at every residue mod 3 of the boundary, in a batch small
    enough for the warp Huffman stage.  The neighbour decodes to its exact bytes, the first unit reports its exact size on
    overflow, and nothing is written outside a region."""
    import torch
    import unarchive_cases as U
    from swcompression_b200 import _lib
    rng = random.Random(144)
    head, tail = H.textlike(300, 145), H.textlike(2000, 146)
    units, caps, expect = [], [], []
    for rep in range(12):
        for d in (1, 2, 5):
            lits = bytes(rng.randrange(256) for _ in range(d))
            cut = U.gzip_member(head) + U.gzip_member(tail)                   # out_cap ends d bytes into the second member
            tiny = U.gzip_member(lits) + U.gzip_member(tail)                  # the first member decodes to d bytes
            for first, cap in ((cut, len(head) + d), (tiny, d + len(tail))):
                nb = U.gzip_member(H.textlike(900 + rep, 147 + rep)) + U.gzip_member(bytes(rng.randrange(256) for _ in range(600)))
                units += [first, nb]
                caps += [cap, len(G.expect(oracle, nb)[1])]
                expect += [G.expect(oracle, first), G.expect(oracle, nb)]
    n = len(units)
    out_off, pos = np.zeros(n, dtype=np.uint64), H.GUARD
    for i in range(n):
        if i % 2 == 0:
            pos += (i // 2) % 3 + 1                         # the boundary behind unit i at every residue mod 3
        out_off[i] = pos
        pos += caps[i]                                      # the next region starts right behind this one
    out_cap = np.array(caps, dtype=np.uint64)
    total = pos + H.GUARD
    buf, offs, lens = H.pack_hostile(units, rng)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_ln, d_used = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(2))
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    keep = [_dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)]
    st = _lib.lib().swc_gzip_multi_unarchive_batch(
        *[_p(t) for t in keep[:3]], _p(d_out), _p(keep[3]), _p(keep[4]), _p(d_ln), _p(d_used), _p(d_st), None, None, None, None,
        None, None, n, 0, None, 0, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    assert H.fence_violations(out, out_off, out_cap).size == 0
    sts, lns = d_st.cpu().numpy(), d_ln.cpu().numpy()
    for i, e in enumerate(expect):
        assert e[0] == G.OK, i
        if out_cap[i] < len(e[1]):
            assert (int(sts[i]), int(lns[i])) == (OVERFLOW, len(e[1])), i
        else:
            got = bytes(out[int(out_off[i]):int(out_off[i]) + int(lns[i])])
            assert (int(sts[i]), got) == (e[0], e[1]), i
