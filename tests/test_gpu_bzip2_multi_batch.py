"""The block-parallel multi-stream BZip2 batch (swc_bzip2_multi_decompress_batch, Batch codec 'bzip2_multi') against the
oracle's BZip2.multiDecompress and the single call swc_bzip2_multi_decompress: the catalogue of tests/bzip2_multi_cases.py
and the byte cuts of its three-stream file, pbzip2-shaped files, a mixed batch, block tables and scratch sizes, overflow and
rerun, a short stream table, fenced hostile layouts, a CUDA-graph replay, Batch.streams and a pbzip2 .tar.bz2 walked in
place."""
import bz2
import ctypes as C
import io
import random
import tarfile

import numpy as np
import pytest

import bzip2_multi_cases as M
import helpers as H

pytestmark = pytest.mark.gpu
OK, OVERFLOW, UNSUPPORTED, WRONG_CRC = 0, 1, 6, 210


@pytest.fixture(scope="module")
def S():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def _cap(oracle, data):
    st, whole, _, _ = M.expect(oracle, data)
    return len(whole) + 64 if st in (OK, WRONG_CRC) else 4 * len(data) + 4096


def _run(units, caps, **kw):
    from swcompression_b200.batch import Batch
    b = Batch.from_units("bzip2_multi", units, np.asarray(caps, dtype=np.uint64), **kw)
    b.run()
    return b


def _answers(b):
    st, ln, used = b.results()
    assert (used == 0).all()
    outs = b.outputs()
    return [(int(st[i]), outs[i], *b.stream_table(i)) for i in range(b.n)]


def _oracle_differences(oracle, units, got, cut_from=None):
    """units whose status, bytes or stream table differ from the oracle's; from unit `cut_from` on (byte cuts), a cut that
    leaves an over-subscribed code set may report SWC_ERR_UNSUPPORTED where the oracle fails otherwise (DESIGN §6)"""
    bad = []
    for i, u in enumerate(units):
        want = M.expect(oracle, u)
        st = got[i][0]
        if cut_from is not None and i >= cut_from and st == UNSUPPORTED and want[0] not in (OK, WRONG_CRC):
            continue
        if st != want[0] or (st in (OK, WRONG_CRC) and tuple(got[i][1:]) != tuple(want[1:])):
            bad.append((i, st, want[0]))
    return bad


def _single(S, data):
    """swc_bzip2_multi_decompress: (status, bytes, stream ends)"""
    L = S._lib.lib()
    buf, n = S._lib.inbuf(data)
    out, out_len, ends, cnt = C.c_void_p(), C.c_size_t(0), C.c_void_p(), C.c_size_t(0)
    st = L.swc_bzip2_multi_decompress(buf, n, C.byref(out), C.byref(out_len), C.byref(ends), C.byref(cnt))
    return st, S._lib.take(out, out_len), list(S._lib.take_sizes(ends, cnt))


def test_catalogue_and_cuts(S, oracle):
    """every case and every byte cut of the three-stream file: the oracle's status, bytes, stream ends and starts; the
    single call's status (on the deviation of DESIGN §6 too), and on OK its bytes and stream ends"""
    units = [c.data for c in M.cases()] + [d for _, d in M.cuts()]
    caps = [_cap(oracle, u) for u in units]
    got = _answers(_run(units, caps))
    assert not _oracle_differences(oracle, units, got, cut_from=len(M.cases()))
    for i, u in enumerate(units):
        st, out, ends = _single(S, u)
        assert st == got[i][0], (i, st, got[i][0])
        if st == OK:
            assert out == got[i][1] and ends == got[i][2]
    names = [c.name for c in M.cases()]
    assert got[names.index("three_hundred_streams")][0] == OK and len(got[names.index("three_hundred_streams")][2]) == 300


def _pbzip2(data, piece=900_000, level=9):
    return b"".join(bz2.compress(data[i:i + piece], level) for i in range(0, len(data), piece)) or bz2.compress(b"", level)


def test_pbzip2_shapes_run_block_parallel(S, oracle):
    """pbzip2-shaped files and `cat`s of multi-block streams: every stream comes from the block stage"""
    raws = [H.textlike(2_500_000 + 100_000 * i, 500 + i) for i in range(3)]
    units = [_pbzip2(r) for r in raws] + [bz2.compress(raws[0][:700_000], 1) + bz2.compress(raws[1][:1_200_000], 2)]
    wants = raws + [raws[0][:700_000] + raws[1][:1_200_000]]
    b = _run(units, [len(w) for w in wants])
    st, ln, _ = b.results()
    par = b.parallel_streams()
    for i, w in enumerate(wants):
        ends, starts = b.stream_table(i)
        assert st[i] == OK and b.output(i) == w
        assert par[i] == len(ends) >= 2
        assert starts == M.expect(oracle, units[i])[3]


def test_mixed_batch_and_table_sizes(S, oracle):
    """clean, damaged and non-bzip2 units side by side; block tables of 1, a few, exactly enough and library-counted, with
    caller scratch and with the pool, give the same answers"""
    from swcompression_b200.batch import Batch
    rng = random.Random(7)
    cases = M.cases()
    units = [c.data for c in cases] + [H.random_bytes(rng, 300), b"BZh9" + H.random_bytes(rng, 200), b"PK\x03\x04"]
    caps = [_cap(oracle, u) for u in units]
    ref = _answers(_run(units, caps))
    assert not _oracle_differences(oracle, units, ref)
    L = S._lib.lib()
    exact = sum(bytes(u).count(bytes.fromhex("314159265359")) for u in units) + 64     # a loose bound of the candidates
    for mb in (1, 5, exact, None):
        for scratch in (None, "sized"):
            kw = dict(max_blocks=mb)
            if scratch:
                kw["scratch_bytes"] = L.swc_bzip2_stream_batch_scratch_bytes(len(units), mb or 0, sum((c + 15) // 16 * 16 for c in caps))
            assert _answers(_run(units, caps, **kw)) == ref, (mb, scratch)


def test_one_slot_scratch(S, oracle):
    units = [_pbzip2(H.textlike(2_000_000, 61), 300_000)] + [c.data for c in M.cases()[:12]]
    caps = [_cap(oracle, u) for u in units]
    ref = _answers(_run(units, caps))
    L = S._lib.lib()
    slot = L.swc_bzip2_stream_batch_scratch_bytes(1, 2, 0) - L.swc_bzip2_stream_batch_scratch_bytes(1, 1, 0)
    fb = L.swc_bzip2_stream_batch_scratch_bytes(len(units), 1, sum((c + 15) // 16 * 16 for c in caps))
    assert _answers(_run(units, caps, max_blocks=64, scratch_bytes=fb + slot)) == ref


def test_overflow_then_rerun(S, oracle):
    """a capacity short by one: overflow with out_len past the capacity; a validated unit reports its exact size, and a
    rerun at out_len is final"""
    raw = H.textlike(1_500_000, 71)
    units = [_pbzip2(raw, 400_000), M.cases()[2].data, b"".join(M.cases()[x].data for x in (3, 4))]
    wants = [M.expect(oracle, u)[1] for u in units]
    b = _run(units, [len(w) - 1 for w in wants])
    st, ln, _ = b.results()
    assert (st == OVERFLOW).all() and (ln > np.array([len(w) - 1 for w in wants])).all()
    assert int(ln[0]) == len(wants[0])
    b2 = _run(units, [int(x) for x in ln])
    st2, ln2, _ = b2.results()
    assert (st2 == OK).all() and b2.outputs() == wants


def test_short_stream_table(S, oracle):
    """a stream table shorter than the stream count: n_streams still counts every stream, the first entries are written"""
    data = b"".join(bz2.compress(H.textlike(1000 + i, 80 + i), 9) for i in range(10))
    b = _run([data, data], [12000 * 2, 12000 * 2], stream_cap=[3, 10])
    st, ln, _ = b.results()
    assert (st == OK).all() and b.d_n_streams.cpu().tolist() == [10, 10]
    want = M.expect(oracle, data)
    assert b.stream_table(0) == (want[2][:3], want[3][:3]) and b.stream_table(1) == (want[2], want[3])


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()


def test_hostile_layout(S, oracle):
    """units at every start residue and back to back, a cut file followed by its own rest, capacities exact, short and
    long between sentinel bytes that must stay intact"""
    import torch
    full = [c.data for c in M.cases() if c.status == OK and c.data][:10] + [_pbzip2(H.textlike(600_000, 95), 200_000)]
    units, tails = [], []
    for i, f in enumerate(full):
        cut = len(f) // 2 if i % 3 == 2 else len(f)
        units.append(f[:cut])
        tails.append(f[cut:] or None)
    sizes = [len(M.expect(oracle, u)[1]) if M.expect(oracle, u)[0] in (OK, WRONG_CRC) else None for u in units]
    out_off, out_cap, total = H.fenced_layout(sizes, 1 << 17)
    buf, offs, lens = H.pack_hostile(units, random.Random(96), None, tails)
    n = len(units)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_len, d_st = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    L = S._lib.lib()
    p = lambda t: C.c_void_p(t.data_ptr())
    d_in, d_off, d_lens, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    st = L.swc_bzip2_multi_decompress_batch(p(d_in), p(d_off), p(d_lens), p(d_out), p(d_oo), p(d_oc), p(d_len), p(d_st),
                                            None, None, None, None, None, None, n, 0, None, 0, stream)
    assert st == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    assert H.fence_violations(out, out_off, out_cap).size == 0
    ln, sts = d_len.cpu().numpy(), d_st.cpu().numpy()
    for i, u in enumerate(units):
        want = M.expect(oracle, u)
        if want[0] in (OK, WRONG_CRC) and len(want[1]) > int(out_cap[i]):
            assert sts[i] == OVERFLOW and ln[i] > out_cap[i]
        else:
            assert sts[i] == want[0], (i, sts[i], want[0])
            if want[0] in (OK, WRONG_CRC):
                assert bytes(out[int(out_off[i]):int(out_off[i]) + int(ln[i])]) == want[1]


def test_graph_replay(S):
    """caller scratch and max_blocks > 0: captured into a CUDA graph, a replay gives the direct call's results"""
    import torch
    units = [_pbzip2(H.textlike(1_000_000, 100 + i), 250_000) for i in range(3)]
    caps = [1_000_000] * 3
    direct = _answers(_run(units, caps, max_blocks=64))
    from swcompression_b200.batch import Batch
    b = Batch.from_units("bzip2_multi", units, np.asarray(caps, dtype=np.uint64), max_blocks=64)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b.run()                                          # warm-up (first-launch constants)
    torch.cuda.synchronize()
    b.d_status.fill_(-1)
    b.d_out.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b.run()
    torch.cuda.synchronize()
    b.d_status.fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    assert _answers(b) == direct


def test_streams_equal_multidecompress(S, oracle):
    """Batch.streams(i) returns what BZip2.multiDecompress returns, or raises its error with its payload"""
    from swcompression_b200 import BZip2
    units = [c.data for c in M.cases()]
    b = _run(units, [_cap(oracle, u) for u in units])
    for i, u in enumerate(units):
        try:
            want = BZip2.multiDecompress(u)
        except Exception as e:                           # noqa: BLE001 - the same error, payload included
            with pytest.raises(type(e)) as got:
                b.streams(i)
            assert got.value.code == e.code and got.value.payload == e.payload
        else:
            assert b.streams(i) == want


def test_tar_of_pbzip2_tar_bz2(S):
    """a pbzip2-shaped .tar.bz2 built with tarfile is walked in place, as TarContainer.info walks the raw tar"""
    from swcompression_b200 import TarContainer
    from swcompression_b200.batch import Batch
    tars = []
    for k in range(2):
        f = io.BytesIO()
        with tarfile.open(fileobj=f, mode="w", format=tarfile.PAX_FORMAT) as t:
            for j in range(6):
                data = H.textlike(300_000 + 50_000 * j, 10 * k + j)
                ti = tarfile.TarInfo(f"dir{k}/file{j}.txt")
                ti.size, ti.mtime = len(data), 1_700_000_000
                t.addfile(ti, io.BytesIO(data))
        tars.append(f.getvalue())
    units = [_pbzip2(t, 900_000) for t in tars]
    b = _run(units, [len(t) for t in tars])
    st, _, _ = b.results()
    assert (st == OK).all() and (b.parallel_streams() >= 2).all()
    w = Batch.tar_of(b)
    w.run()
    for i, t in enumerate(tars):
        assert [e.name for e in w.entries(i)] == [e.name for e in TarContainer.info(t)]
        assert [e.size for e in w.entries(i)] == [e.size for e in TarContainer.info(t)]
