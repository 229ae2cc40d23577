"""The batched LZ4 frame decoder (swc_lz4_frame_decompress_batch, swc_lz4_frame_info_batch) against the writer's model of
LZ4.decompress(data:dictionary:dictionaryID:) and against swc_lz4_decompress on the same bytes: status, out_len, consumed
bytes and bytes unit by unit on the catalogue of tests/lz4_frame_cases.py and every byte cut of its small cases, mixed and
hostile layouts, output overflow and rerun, a block table that is too small, the raw block batch, a CUDA-graph capture."""
import ctypes as C
import random

import numpy as np
import pytest

import helpers as H
import lz4_frame_cases as F
import lz4_writer as W
from lz4_writer import FBlock

pytestmark = pytest.mark.gpu
OVERFLOW, UNSUPPORTED = 1, 6


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


def _infos(buf, offs, lens, dictionary=None, dict_id=None):
    import torch
    from swcompression_b200 import _lib
    n = len(offs)
    size = C.sizeof(_lib.Lz4FrameInfo)
    d_info = torch.zeros(max(n, 1) * size, dtype=torch.uint8, device="cuda")
    d_in, d_off, d_len = _dev(buf), _dev(offs), _dev(lens)
    assert _lib.lib().swc_lz4_frame_info_batch(_p(d_in), _p(d_off), _p(d_len), dictionary is not None, dict_id is not None,
                                               dict_id or 0, _p(d_info), n, _stream()) == 0
    torch.cuda.synchronize()
    raw = d_info.cpu().numpy().tobytes()
    return [_lib.Lz4FrameInfo.from_buffer_copy(raw, i * size) for i in range(n)]


def _exact_blocks(units, dictionary=None, dict_id=None):
    from swcompression_b200.batch import pack_units
    buf, offs, lens = pack_units(units)
    return max(1, sum(i.n_blocks for i in _infos(buf, offs, lens, dictionary, dict_id)))


def _run(units, caps, dictionary=None, dict_id=None, max_blocks=None):
    from swcompression_b200.batch import Batch
    b = Batch.from_units("lz4_frame", units, caps, aux=dictionary, dict_id=dict_id, max_blocks=max_blocks)
    b.run()
    st, ln, used = b.results()
    return b, st, ln, used, b.outputs()


def _single(data, dictionary=None, dict_id=None):
    from swcompression_b200 import _lib
    buf, n = _lib.inbuf(data)
    dbuf, dn = _lib.inbuf(dictionary) if dictionary is not None else (None, 0)
    out, ol, used = C.c_void_p(), C.c_size_t(), C.c_size_t()
    st = _lib.lib().swc_lz4_decompress(buf, n, dbuf, dn, dict_id is not None, dict_id or 0, C.byref(out), C.byref(ol), C.byref(used))
    return st, _lib.take(out, ol), used.value


def _compare(cases, st, ln, used, outs):
    bad = []
    for i, c in enumerate(cases):
        if st[i] != c.status:
            bad.append((c.name, "status", int(st[i]), c.status))
        elif ln[i] != len(c.out) or outs[i] != c.out or used[i] != c.consumed:
            bad.append((c.name, "len/bytes/consumed", int(ln[i]), len(c.out), int(used[i]), c.consumed))
    return bad


def _groups(cases):
    groups = {}
    for c in cases:
        groups.setdefault(c.key, []).append(c)
    return groups


def test_catalogue(S):
    """every case, grouped by the dictionary and ID it is decoded with: once with the library counting the blocks, once with
    an exact max_blocks and caller scratch; and swc_lz4_decompress on the same bytes"""
    cases = F.catalogue()
    assert sum(c.dictionary is not None for c in cases) > 100 and sum(c.dict_id is not None for c in cases) >= 4
    for (d, did), group in _groups(cases).items():
        units = [c.data for c in group]
        caps = np.array([len(c.out) for c in group], dtype=np.uint64)          # failures need no room at all
        for max_blocks in (None, _exact_blocks(units, d, did)):
            _, st, ln, used, outs = _run(units, caps, d, did, max_blocks)
            bad = _compare(group, st, ln, used, outs)
            assert not bad, (len(bad), len(group), max_blocks, bad[:8])
    for c in cases:
        if len(c.data) < 200000:
            sst, sout, sused = _single(c.data, c.dictionary, c.dict_id)
            assert sst == c.status and (sst not in F.PAYLOAD or (sout == c.out and sused == c.consumed)), c.name


def test_truncations(S):
    """every byte cut of every case of at most 400 bytes, the rest of the stream lying behind the unit in memory"""
    from swcompression_b200.batch import Batch
    cuts = F.truncations()
    total = 0
    for (d, did), group in _groups([c for c, _ in cuts]).items():
        tails = {id(c): t for c, t in cuts}
        buf, offs, lens = H.pack_hostile([c.data for c in group], random.Random(71), None, [tails[id(c)] for c in group])
        caps = np.array([len(c.out) for c in group], dtype=np.uint64)
        for max_blocks in (None, max(1, sum(i.n_blocks for i in _infos(buf, offs, lens, d, did)))):
            b = Batch("lz4_frame", buf, offs, lens, caps, aux=d, dict_id=did, max_blocks=max_blocks)
            b.run()
            st, ln, used = b.results()
            bad = _compare(group, st, ln, used, b.outputs())
            assert not bad, (len(bad), len(group), bad[:8])
        total += len(group)
        for i in random.Random(72).sample(range(len(group)), min(300, len(group))):
            assert _single(group[i].data, d, did)[0] == st[i], group[i].name
    assert total > 10000


def test_mixed_batch(S):
    """a few thousand units of all three kinds, failing ones between sound ones, shuffled"""
    pool = [c for c in F.catalogue() if c.dictionary is None and c.dict_id is None and len(c.data) < 20000]
    assert {c.kind for c in pool} >= {F.INDEPENDENT, F.DEPENDENT, F.LEGACY}
    rng = random.Random(73)
    cases = [pool[rng.randrange(len(pool))] for _ in range(4000)]
    assert sum(c.status != 0 for c in cases) > 300 and sum(c.status == 0 for c in cases) > 300
    _, st, ln, used, outs = _run([c.data for c in cases], np.array([len(c.out) for c in cases], dtype=np.uint64))
    assert not _compare(cases, st, ln, used, outs)


def _hostile(cases, tails, rng, aligned):
    import torch
    from swcompression_b200 import _lib
    sizes = [len(c.out) if c.status in F.PAYLOAD else None for c in cases]
    out_off, out_cap, total = H.fenced_layout(sizes, 64)
    buf, offs, lens = H.pack_hostile([c.data for c in cases], rng, None, tails, residues=[0] * len(cases) if aligned else None)
    n = len(cases)
    d_in, d_off, d_len, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_ln = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_used = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    assert _lib.lib().swc_lz4_frame_decompress_batch(_p(d_in), _p(d_off), _p(d_len), None, 0, 0, 0, _p(d_out), _p(d_oo), _p(d_oc),
                                                     _p(d_ln), _p(d_used), _p(d_st), n, 0, None, 0, _stream()) == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    outs = [bytes(out[int(o):int(o) + int(c)]) for o, c in zip(out_off, out_cap)]
    return d_st.cpu().numpy(), d_ln.cpu().numpy(), d_used.cpu().numpy(), outs, out_cap, H.fence_violations(out, out_off, out_cap)


def test_hostile_layout(S):
    """units at all 16 start residues and back to back, cut frames followed by their own rest, capacities exact, 1-15 short
    and 1-15 long between sentinel bytes that must stay intact; the aligned packing gives the same statuses"""
    rng = random.Random(74)
    whole = [c for c in F.catalogue() if c.dictionary is None and c.dict_id is None and 0 < len(c.data) < 20000]
    cases, tails = [], []
    for j in range(600):
        c = whole[rng.randrange(len(whole))]
        if j % 3 == 2:                                  # the layout gives every unit with j % 3 == 1 a short region
            k = rng.randrange(1, len(c.data))
            cases.append(F.FCase(f"{c.name}[:{k}]", c.data[:k])); tails.append(c.data[k:])
        else:
            cases.append(c); tails.append(W.frame([FBlock(F.cblock(1))]) if j % 2 else None)
    st, ln, used, outs, caps, fence = _hostile(cases, tails, rng, False)
    bad = []
    for i, c in enumerate(cases):
        if c.status in F.PAYLOAD and len(c.out) > caps[i]:
            if st[i] != OVERFLOW or ln[i] != len(c.out) or used[i] != 0:
                bad.append((c.name, "overflow", int(st[i]), int(ln[i]), len(c.out)))
        elif st[i] != c.status or ln[i] != len(c.out) or used[i] != c.consumed or outs[i][:len(c.out)] != c.out:
            bad.append((c.name, int(st[i]), c.status, int(ln[i]), len(c.out)))
    assert not bad and fence.size == 0, (bad[:8], fence[:8])
    assert (st == OVERFLOW).sum() > 20
    st2, ln2, used2, _, _, fence2 = _hostile(cases, tails, random.Random(74), True)
    assert (st2 == st).all() and (ln2 == ln).all() and (used2 == used).all() and fence2.size == 0


def test_output_overflow_then_rerun(S):
    """capacity one short at every block boundary of a multi-block frame (all three kinds, and a checksumMismatch unit): the
    unit reports the exact size; the rerun with out_len gives the model's answer.  A unit that fails
    behind the boundary reports its failure, not the overflow."""
    blocks = F.mixed_blocks(40)
    want = W.decode(W.frame(blocks)).out
    streams = [W.frame(blocks, independent=True, block_checksums=True), W.frame(blocks), W.legacy_frame([F.cblock(j) for j in range(40)]),
               W.frame(blocks, independent=True, content_checksum=want + b"x"), W.frame(blocks, content_checksum=want + b"x"),
               W.frame(blocks[:39] + [FBlock(F.cblock(39)[:-3])], independent=True), W.frame(blocks[:39] + [FBlock(F.cblock(39)[:-3])])]
    cases, caps = [], []
    for s in streams:
        c = F.FCase("o", s)
        sizes = np.cumsum([len(W.decode_block(b.data).out) if not b.stored else len(b.data) for b in blocks])
        for edge in sorted(set(int(x) for x in sizes)):
            cases.append(c); caps.append(max(edge - 1, 0))
    _, st, ln, used, outs = _run([c.data for c in cases], np.array(caps, dtype=np.uint64))
    for i, c in enumerate(cases):
        if c.status in F.PAYLOAD and caps[i] < len(c.out):
            assert st[i] == OVERFLOW and ln[i] == len(c.out) and used[i] == 0, (i, c.status, int(st[i]), int(ln[i]))
        else:
            assert st[i] == c.status, (i, c.status, int(st[i]))
    assert (st == OVERFLOW).sum() > 150 and (st == W.TRUNCATED).sum() > 50
    redo = [i for i in range(len(cases)) if st[i] == OVERFLOW]
    _, st2, ln2, used2, outs2 = _run([cases[i].data for i in redo], ln[redo].astype(np.uint64))
    assert not _compare([cases[i] for i in redo], st2, ln2, used2, outs2)
    assert (st2 == W.CHECKSUM).sum() > 50


def test_block_table_too_small(S):
    """units are placed in order: those that fit are right, the rest report SWC_ERR_UNSUPPORTED and write nothing; a unit
    without blocks always fits"""
    import torch
    mk = lambda nb, ind: F.FCase("t", W.frame(F.mixed_blocks(nb), independent=ind))
    cases = [mk(10, True), mk(20, False), F.FCase("t", W.legacy_frame([F.cblock(1)] * 5)), mk(40, True), mk(3, False), mk(0, True),
             F.FCase("t", b"\x04\x22\x4D"), mk(2, True)]
    from swcompression_b200.batch import Batch
    b = Batch.from_units("lz4_frame", [c.data for c in cases], np.array([len(c.out) for c in cases], dtype=np.uint64), max_blocks=36)
    b.d_out.fill_(H.SENTINEL)
    b.run()
    st, ln, used = b.results()
    outs = b.outputs()
    assert not _compare(cases[:3] + cases[5:7], list(st[:3]) + list(st[5:7]), list(ln[:3]) + list(ln[5:7]),
                        list(used[:3]) + list(used[5:7]), outs[:3] + outs[5:7])
    host = b.d_out.cpu().numpy()
    for i in (3, 4, 7):
        o = int(b.h_out_off[i])
        assert st[i] == UNSUPPORTED and ln[i] == 0 and used[i] == 0 and (host[o:o + len(cases[i].out)] == H.SENTINEL).all(), i


def test_equals_raw_block_batch(S):
    """the blocks of independent frames through swc_lz4_block_decompress_batch give the same bytes"""
    from swcompression_b200.batch import Batch
    raws = [H.textlike(3000 + 977 * k, 800 + k) for k in range(24)]
    comp = [H.lz4_block_compress(r) for r in raws]
    frames = [W.frame([FBlock(comp[(f + j) % 24]) for j in range(1 + f % 7)], independent=True, block_checksums=f % 2 == 0, bd=0x40)
              for f in range(50)]
    want = [b"".join(raws[(f + j) % 24] for j in range(1 + f % 7)) for f in range(50)]
    _, st, ln, used, outs = _run(frames, np.array([len(w) for w in want], dtype=np.uint64))
    assert (st == 0).all() and outs == want and list(used) == [len(f) for f in frames]
    r = Batch.from_units("lz4_block", comp, 40000)
    r.run()
    assert (r.results()[0] == 0).all() and r.outputs() == raws


def test_graph_capture(S):
    """with caller scratch and max_blocks > 0 the call reads nothing back and allocates nothing: captured into a CUDA graph,
    the results stay untouched until the replay, then equal the eager run's"""
    import torch
    from swcompression_b200.batch import Batch
    cases = [c for c in F.catalogue() if c.dictionary is F.DICT and c.dict_id is None and len(c.data) < 50000][:200]
    cases += [c for c in F.catalogue() if c.name.startswith(("ind_", "legacy", "dep ", "ind "))][:150]
    cases = [F.FCase(c.name, c.data, F.DICT) for c in cases]
    units = [c.data for c in cases]
    b = Batch.from_units("lz4_frame", units, np.array([len(c.out) for c in cases], dtype=np.uint64), aux=F.DICT,
                         max_blocks=_exact_blocks(units, F.DICT) + 7)
    b.run()
    st0, ln0, used0 = b.results()
    outs0 = b.outputs()
    assert not _compare(cases, st0, ln0, used0, outs0)
    b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_consumed.zero_(); b.d_out.zero_()
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
    assert (st1 == st0).all() and (ln1 == ln0).all() and (used1 == used0).all() and b.outputs() == outs0


def test_frame_info(S):
    """swc_lz4_frame_info_batch against the writer's own knowledge of each case"""
    from swcompression_b200.batch import pack_units
    cases = [c for c in F.catalogue() if c.dictionary is None and c.dict_id is None]
    infos = _infos(*pack_units([c.data for c in cases]))
    checked = 0
    for c, i in zip(cases, infos):
        if c.kind is not None and i.kind != F.NONE:
            assert i.kind == c.kind and c.n_blocks in (None, i.n_blocks), (c.name, i.kind, i.n_blocks)
            checked += 1
        if c.status in F.PAYLOAD:
            assert i.status == 0 and i.frame_end == c.consumed and i.kind != F.NONE, c.name
        if i.kind == F.NONE:
            assert i.status == c.status and i.n_blocks == 0, c.name
    assert checked > 500
    by = {c.name: i for c, i in zip(cases, infos)}
    assert by["skip one"].frame_start == 11 and by["skip one"].flags & 0x100
    sized = by["dep 5 blocks size right"]
    assert sized.content_size == len(W.decode(W.frame(F.mixed_blocks(5))).out) and by["skip one"].content_size == 2 ** 64 - 1
    assert by["dep 5 blocks checksum missing"].flags & 0x200 and by["dep 5 blocks checksum missing"].status == W.TRUNCATED
    assert by["bd 0x50 stored block of max+1 ind"].status == W.CORRUPTED and by["bd 0x50 stored block of max ind"].max_block_size == 256 << 10


def test_roundtrip_compress(S):
    """frames written by LZ4.compress for every option combination decode to their input"""
    from swcompression_b200 import _lib
    data = H.textlike(150000, 77)
    d = F.DICT
    for use_dict in (False, True):
        frames = []
        for opt in range(32):
            ind, bck, cck, csz, did = (opt >> k & 1 for k in range(5))
            if did and not use_dict:
                continue
            buf, n = _lib.inbuf(data)
            dbuf, dn = _lib.inbuf(d) if use_dict else (None, 0)
            out, ol = C.c_void_p(), C.c_size_t()
            assert _lib.lib().swc_lz4_compress(buf, n, ind, bck, cck, csz, 65536 if opt % 3 else 40000, dbuf, dn, did, 9,
                                               C.byref(out), C.byref(ol)) == 0
            frames.append(_lib.take(out, ol))
        _, st, ln, used, outs = _run(frames, len(data), d if use_dict else None, 9 if use_dict else None)
        assert (st == 0).all() and all(o == data for o in outs) and list(used) == [len(f) for f in frames]
