"""swc_gzip_archive_batch / swc_zlib_archive_batch (archive_compress.cu) byte for byte against the CPU restatement of
GzipArchive.archive and ZlibArchive.archive, and back through the engine's own unarchive batches: the Deflate catalogue
with a header per unit, hostile input and output layouts with capacity fences, slices of the scratch, the max_in_bytes
bound, a CUDA-graph capture, the single calls as one-unit batches and the benched shape."""
import ctypes as C
import random

import numpy as np
import pytest

import archive_options as AO
import compress_batch as CB
import deflatec_cases as K
import helpers as H

pytestmark = pytest.mark.gpu
OK, OVERFLOW, INVALID_ARG, UNSUPPORTED = 0, 1, 4, 6


@pytest.fixture(scope="module")
def oc():
    import swco_deflatec
    swco_deflatec.lib()
    return swco_deflatec


@pytest.fixture(scope="module")
def S():
    import torch
    assert torch.cuda.is_available()
    import swcompression_b200 as S
    return S


def expected(oc, kind, units, opts):
    if kind == "zlib":
        return [oc.zlib_archive(u)[1] for u in units]
    return [oc.gzip_archive(u, **AO.oracle_keywords(o))[1] for u, o in zip(units, opts)]


def header_cols(opts):
    """per-unit headers packed back to back (identical ones once) -> (blob, offsets, lengths)"""
    from swcompression_b200 import GzipArchive
    blob, at = bytearray(), {}
    off, ln = np.zeros(len(opts), dtype=np.uint64), np.zeros(len(opts), dtype=np.uint64)
    for i, o in enumerate(opts):
        h = GzipArchive.archive_header(**o)
        if h not in at:
            at[h] = len(blob)
            blob += h
        off[i], ln[i] = at[h], len(h)
    return bytes(blob), off, ln


def run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, max_in=0, scratch=-1):
    """-> (return code, status, out_len, output buffer); scratch -1: swc_archive_compress_batch_scratch_bytes of the
    batch, None: the library pool"""
    import torch
    from swcompression_b200 import _lib
    L = _lib.lib()
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to(dev)
    n = len(in_off)
    d_in = torch.from_numpy(np.ascontiguousarray(in_buf)).to(dev)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device=dev)
    d_len, d_st = torch.zeros(n, dtype=torch.int64, device=dev), torch.full((n,), -1, dtype=torch.int32, device=dev)
    if scratch == -1:
        scratch = L.swc_archive_compress_batch_scratch_bytes(n, max_in or int(np.asarray(in_len, dtype=np.uint64).sum()))
    scr = None if scratch is None else torch.empty(max(scratch, 1), dtype=torch.uint8, device=dev)
    p = lambda x: C.c_void_p(x.data_ptr())
    s = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    sp, sb = (None, 0) if scr is None else (p(scr), scratch)
    i_off, i_len, o_off, o_cap = t(in_off), t(in_len), t(out_off), t(out_cap)
    if kind == "gzip":
        blob, h_off, h_len = header_cols(opts)
        d_h = torch.from_numpy(np.frombuffer(blob + b"\0", dtype=np.uint8).copy()).to(dev)
        d_ho, d_hl = t(h_off), t(h_len)
        rc = L.swc_gzip_archive_batch(p(d_in), p(i_off), p(i_len), p(d_h), p(d_ho), p(d_hl), p(d_out), p(o_off), p(o_cap),
                                      p(d_len), p(d_st), n, max_in, sp, sb, s)
    else:
        rc = L.swc_zlib_archive_batch(p(d_in), p(i_off), p(i_len), p(d_out), p(o_off), p(o_cap), p(d_len), p(d_st), n, max_in,
                                      sp, sb, s)
    torch.cuda.synchronize()
    return rc, d_st.cpu().numpy(), d_len.cpu().numpy(), d_out.cpu().numpy()


def check_fenced(st, ln, out, exp, out_off, out_cap, skip=()):
    """every unit exact or overflowing with its exact size, nothing written outside the units that succeed"""
    written = np.zeros(len(out), dtype=bool)
    for j, e in enumerate(exp):
        if j in skip:
            continue
        o = int(out_off[j])
        assert ln[j] == len(e), j
        if out_cap[j] < len(e):
            assert st[j] == OVERFLOW, j
        else:
            assert st[j] == OK and bytes(out[o:o + len(e)]) == e, j
            written[o:o + len(e)] = True
    return written


def catalogue_units():
    return [d for _, d in K.cases()] + list(CB.mixed_units())


def cycled_opts(n):
    grid = [api for api, _ in AO.grid()]
    return [grid[i % len(grid)] for i in range(n)]


@pytest.mark.parametrize("kind", ["gzip", "zlib"])
def test_catalogue_and_round_trip(S, oc, kind):
    """1 and 2: every catalogue unit, gzip with its own header, equals the oracle's archive and decodes back through the
    engine's unarchive batch with consumed == out_len"""
    from swcompression_b200.batch import Batch
    units = catalogue_units()
    opts = cycled_opts(len(units)) if kind == "gzip" else None
    caps = [S.GzipArchive.max_archive_size(len(u), **o) for u, o in zip(units, opts)] if opts else \
        [S.ZlibArchive.max_archive_size(len(u)) for u in units]
    b = Batch.from_units(kind + "_archive", units, caps, gzip_options=opts)
    b.run()
    st, ln, _ = b.results()
    outs = b.outputs()
    exp = expected(oc, kind, units, opts)
    for j, e in enumerate(exp):
        assert st[j] == OK and ln[j] == len(e) and outs[j] == e, j
    d = Batch.from_units(kind, outs, [max(len(u), 16) for u in units], headers=kind == "gzip")
    d.run()
    dst, dln, used = d.results()
    assert (dst == OK).all() and d.outputs() == units and (used == ln).all()
    if kind == "gzip":
        for j, h in enumerate(d.gzip_headers()):
            o = opts[j]
            assert h.os_type == AO.OS_BYTES[o["osType"]] and h.is_text_file == int(o["isTextFile"]), j
            assert h.has_file_name == (o["fileName"] is not None) and h.has_comment == (o["comment"] is not None), j
            assert h.header_len == len(S.GzipArchive.archive_header(**o)), j
            mt = o["modificationTime"]
            assert h.modification_time == (0 if mt is None else int(mt) & 0xFFFFFFFF), j


@pytest.mark.parametrize("kind", ["gzip", "zlib"])
def test_hostile_layout(S, oc, kind):
    """3: hostile inputs; regions at every start residue with exact, short, long and below-framing capacities.
    Overflowing units report the exact size and write nothing; a rerun at that size gives the archive."""
    units = list(CB.mixed_units())
    opts = cycled_opts(len(units)) if kind == "gzip" else None
    exp = expected(oc, kind, units, opts)
    in_buf, in_off, in_len = H.pack_hostile(units, random.Random(5))
    out_off, out_cap, total = H.fenced_layout([len(e) for e in exp], align=1)
    # every fourth unit below its header + trailer
    frame = [len(e) - len(oc.deflate_compress(u)[1]) for e, u in zip(exp, units)]
    for j in range(3, len(units), 4):
        out_cap[j] = frame[j] - 1 - j % frame[j]
    rc, st, ln, out = run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total)
    assert rc == OK
    written = check_fenced(st, ln, out, exp, out_off, out_cap)
    assert (out[~written] == H.SENTINEL).all()
    assert len(H.fence_violations(out, out_off, out_cap)) == 0
    over = [j for j in range(len(units)) if st[j] == OVERFLOW]
    assert len(over) > len(units) // 4
    # the rerun: every region exactly the reported size, in a layout with room for it
    out_off2, _, total2 = H.fenced_layout([int(x) + 16 for x in ln], align=1)
    rc, st2, ln2, out2 = run(kind, in_buf, in_off, in_len, opts, out_off2, ln.astype(np.uint64), total2)
    assert rc == OK and (st2 == OK).all() and (ln2 == ln).all()
    for j in over:
        o = int(out_off2[j])
        assert bytes(out2[o:o + len(exp[j])]) == exp[j], j


@pytest.mark.parametrize("kind", ["gzip", "zlib"])
def test_slices(S, oc, kind):
    """4: max_in_bytes == 0 with a caller scratch that holds only the largest unit runs in several slices with the same
    results; one below it is invalid; the library pool works"""
    from swcompression_b200 import _lib
    units = list(CB.mixed_units())
    opts = cycled_opts(len(units)) if kind == "gzip" else None
    exp = expected(oc, kind, units, opts)
    in_buf, in_off, in_len = H.pack_hostile(units, random.Random(6))
    out_off, out_cap, total = H.fenced_layout([len(e) for e in exp], align=1)
    L = _lib.lib()
    full = run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total)
    small = L.swc_archive_compress_batch_scratch_bytes(1, int(in_len.max()))
    n0 = L.swc_kernel_launches()
    sliced = run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, scratch=small)
    assert L.swc_kernel_launches() - n0 > 7
    pool = run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, scratch=None)
    for r in (full, sliced, pool):
        assert r[0] == OK
        for x, y in zip(full[1:], r[1:]):
            assert (x == y).all()
    check_fenced(*full[1:], exp, out_off, out_cap)
    # a quarter of the one-unit scratch is below the need of the largest unit
    assert run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, scratch=small // 4)[0] == INVALID_ARG


@pytest.mark.parametrize("kind", ["gzip", "zlib"])
def test_max_in_bytes(S, oc, kind):
    """5: units past max_in_bytes are unsupported with out_len 0 and untouched regions, earlier ones exact; a scratch
    below swc_archive_compress_batch_scratch_bytes is invalid"""
    from swcompression_b200 import _lib
    units = list(CB.mixed_units())
    opts = cycled_opts(len(units)) if kind == "gzip" else None
    exp = expected(oc, kind, units, opts)
    in_buf, in_off, in_len = H.pack_hostile(units, random.Random(7))
    # regions of at least len + 5 bytes; every unit that fits has room
    out_off, _, total = H.fenced_layout([len(e) + 20 for e in exp], align=1)
    out_cap = np.array([len(e) + 3 for e in exp], dtype=np.uint64)
    prefix = np.concatenate([[0], np.cumsum(in_len.astype(np.int64))])
    cut = len(units) // 2
    for max_in in (int(prefix[cut]), int(prefix[cut]) + int(in_len[cut]) - 1 if in_len[cut] else int(prefix[cut])):
        rc, st, ln, out = run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, max_in=max_in)
        assert rc == OK
        fits = [prefix[j] + int(in_len[j]) <= max_in for j in range(len(units))]
        assert fits[cut - 1] and not all(fits)
        written = check_fenced(st, ln, out, exp, out_off, out_cap, skip={j for j, f in enumerate(fits) if not f})
        for j, f in enumerate(fits):
            if not f:
                assert st[j] == UNSUPPORTED and ln[j] == 0, j
        assert (out[~written] == H.SENTINEL).all()
    L = _lib.lib()
    need = L.swc_archive_compress_batch_scratch_bytes(len(units), int(prefix[-1]))
    assert run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, max_in=int(prefix[-1]), scratch=need - 1)[0] == INVALID_ARG
    rc, st, ln, out = run(kind, in_buf, in_off, in_len, opts, out_off, out_cap, total, max_in=int(prefix[-1]), scratch=need)
    assert rc == OK and (st == OK).all()


def test_graph_capture(S, oc):
    """6: with caller scratch and max_in_bytes, a gzip and a zlib batch captured into a CUDA graph; a replay on new bytes
    of the same lengths gives the new bytes' archives"""
    import torch
    from swcompression_b200 import _lib
    from swcompression_b200.batch import Batch, pack_units
    rng = random.Random(13)
    text = H.textlike(300000, 31)
    lens = [0, 1, 2, 700, 4096, 4097, 20000, 65536, 70001, 131075]
    first = [text[:n] for n in lens]
    second = [H.random_bytes(rng, n) if k % 2 else text[::-1][:n] for k, n in enumerate(lens)]
    opts = cycled_opts(len(lens))
    L = _lib.lib()
    batches = []
    for kind in ("gzip", "zlib"):
        o = opts if kind == "gzip" else None
        caps = [S.GzipArchive.max_archive_size(n, **x) for n, x in zip(lens, opts)] if o else \
            [S.ZlibArchive.max_archive_size(n) for n in lens]
        b = Batch.from_units(kind + "_archive", first, caps, gzip_options=o, max_in_bytes=sum(lens))
        n0 = L.swc_kernel_launches()
        b.run()
        assert L.swc_kernel_launches() - n0 == 7
        assert b.outputs() == expected(oc, kind, first, o)
        b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_out.zero_()
        batches.append((kind, o, b))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _, _, b in batches:
                b.run()
    torch.cuda.synchronize()
    buf, _, _ = pack_units(second)
    for _, _, b in batches:
        assert (b.d_status.cpu().numpy() == -1).all()
        b.d_in.copy_(torch.from_numpy(buf).cuda())
    g.replay()
    for kind, o, b in batches:
        st, ln, _ = b.results()
        assert (st == OK).all()
        assert b.outputs() == expected(oc, kind, second, o), kind


def test_single_calls_are_the_one_unit_batch(S, oc):
    """7: GzipArchive.archive / ZlibArchive.archive equal unit 0 of a one-unit batch"""
    from swcompression_b200.batch import Batch
    opts = dict(comment="single", fileName="one.bin", writeHeaderCRC=True, modificationTime=1700000000, osType="unix")
    for data in (H.textlike(64 << 20, 9), bytes(64 << 20)):
        g = S.GzipArchive.archive(data, **opts)
        b = Batch.from_units("gzip_archive", [data], S.GzipArchive.max_archive_size(len(data), **opts), gzip_options=opts)
        b.run()
        assert b.results()[0][0] == OK and b.output(0) == g
        assert g == oc.gzip_archive(data, **AO.oracle_keywords(opts))[1]
        z = S.ZlibArchive.archive(data)
        b = Batch.from_units("zlib_archive", [data], S.ZlibArchive.max_archive_size(len(data)))
        b.run()
        assert b.results()[0][0] == OK and b.output(0) == z
        del b


def benched_units():
    """the 80 / 10 / 10 text / zeros / random mix of 64 KiB units that tools/bench_archive_batch.py tiles"""
    rng = random.Random(4)
    distinct = []
    for i in range(64):
        r = i % 10
        distinct.append(bytes(65536) if r == 8 else H.random_bytes(rng, 65536) if r == 9 else H.textlike(65536, 500 + i))
    return distinct


@pytest.mark.parametrize("kind", ["gzip", "zlib"])
def test_benched_shape(S, oc, kind):
    """8: 20 480 tiled 64 KiB units with max_in_bytes: the first 64 equal the oracle, every tile equals the first"""
    import torch
    from swcompression_b200.batch import Batch
    distinct = benched_units()
    tile = 320
    buf = np.frombuffer(b"".join(distinct) * tile + bytes(64), dtype=np.uint8)
    n = 64 * tile
    offs = np.arange(n, dtype=np.uint64) * np.uint64(65536)
    opts = dict(fileName="member.bin", modificationTime=1700000000)
    cap = S.GzipArchive.max_archive_size(65536, **opts) if kind == "gzip" else S.ZlibArchive.max_archive_size(65536)
    b = Batch(kind + "_archive", buf, offs, np.full(n, 65536, dtype=np.uint64), cap,
              gzip_options=opts if kind == "gzip" else None, max_in_bytes=n * 65536)
    b.d_out.zero_()
    b.run()
    st, ln, _ = b.results()
    assert (st == OK).all() and (ln.reshape(tile, 64) == ln[:64][None, :]).all()
    exp = expected(oc, kind, distinct, [opts] * 64 if kind == "gzip" else None)
    assert [int(x) for x in ln[:64]] == [len(e) for e in exp]
    stride = (cap + 15) // 16 * 16
    out = b.d_out[: n * stride].view(tile, 64, stride)
    assert bool((out == out[0:1]).all())
    host = out[0].cpu().numpy()
    for j, e in enumerate(exp):
        assert bytes(host[j, :len(e)]) == e, j
    del out, b
    torch.cuda.empty_cache()
