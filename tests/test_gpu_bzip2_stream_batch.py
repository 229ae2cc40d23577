"""The block-parallel BZip2 stream batch (swc_bzip2_stream_decompress_batch) against the oracle's BZip2.decompress and
against the one-warp-per-stream batch (swc_bzip2_decompress_batch) on the same bytes and capacities: the hand-built
catalogue of tests/bzip2_cases.py (magics inside payloads, blocks larger than a slot) and its truncations, real multi-block
streams from libbzip2, damage inside them, overflow and rerun, a block table that is too small, one-slot scratch, hostile
layouts with fenced outputs, and a CUDA-graph capture replayed on new inputs."""
import bz2
import ctypes as C
import functools
import random

import numpy as np
import pytest

import bzip2_cases as D
import helpers as H

pytestmark = pytest.mark.gpu
OK, OVERFLOW, UNSUPPORTED, WRONG_CRC = 0, 1, 6, 210
BLOCK_MAGIC, END_MAGIC = format(0x314159265359, "048b"), format(0x177245385090, "048b")


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


def _run(codec, units, caps, **kw):
    from swcompression_b200.batch import Batch
    b = Batch.from_units(codec, units, np.asarray(caps, dtype=np.uint64), **kw)
    b.run()
    st, ln, used = b.results()
    return st, ln, used, b.outputs()


def _both(units, caps, **kw):
    """-> (new batch results, old batch results), each (status, out_len, consumed, outputs)"""
    return _run("bzip2_stream", units, caps, **kw), _run("bzip2", units, caps)


def _differences(new, old):
    """units where the new batch breaks the equality with the old one: the same status; on OK / wrongCRC the same bytes,
    size and consumed bits; on overflow a size at least the old lower bound"""
    bad = []
    for i in range(len(new[0])):
        s, o = int(new[0][i]), int(old[0][i])
        if s != o:
            bad.append((i, "status", s, o))
        elif s in (OK, WRONG_CRC) and (new[1][i] != old[1][i] or new[2][i] != old[2][i] or new[3][i] != old[3][i]):
            bad.append((i, "result", int(new[1][i]), int(old[1][i]), int(new[2][i]), int(old[2][i])))
        elif s == OVERFLOW and new[1][i] < old[1][i]:
            bad.append((i, "overflow size", int(new[1][i]), int(old[1][i])))
    return bad


def _oracle_differences(oracle, units, new):
    bad = []
    for i, u in enumerate(units):
        ost, oout, oused = oracle.bzip2_decompress(u)
        st = int(new[0][i])
        if st != ost or (st in (OK, WRONG_CRC) and new[3][i] != oout) or (st == OK and new[2][i] != oused):
            bad.append((i, st, ost))
    return bad


def _slot_bytes(L):
    # the columns of one and two entries both fit their 256-byte minimum, so the difference is one slot
    return L.swc_bzip2_stream_batch_scratch_bytes(1, 2, 0) - L.swc_bzip2_stream_batch_scratch_bytes(1, 1, 0)


def _magics(stream):
    """bit positions of the block magics and the first end magic (a real stream has no look-alikes)"""
    bits = bin(int.from_bytes(b"\x01" + stream, "big"))[3:]
    blocks, at = [], bits.find(BLOCK_MAGIC)
    while at >= 0:
        blocks.append(at)
        at = bits.find(BLOCK_MAGIC, at + 1)
    return blocks, bits.find(END_MAGIC)


def _flip(stream, bit):
    b = bytearray(stream)
    b[bit // 8] ^= 0x80 >> (bit % 8)
    return bytes(b)


def _insert(stream, bit, junk):
    """`stream` with the bit string `junk` inserted at `bit`, zero bits filling the last byte"""
    bits = bin(int.from_bytes(b"\x01" + stream, "big"))[3:]
    bits = bits[:bit] + junk + bits[bit:]
    bits += "0" * (-len(bits) % 8)
    return int(bits, 2).to_bytes(len(bits) // 8, "big")


def _text(n, seed):
    return H.textlike(n, seed)


def test_catalogue(S, oracle):
    """every hand-built case at the capacity room(c): the status the case declares for the engine, the oracle's bytes and
    consumed bits, and the old batch's answer; once with the library's pool, once with a small table and scratch"""
    cases = D.catalogue()
    units, caps = [c.data for c in cases], [D.room(c) for c in cases]
    assert {"level_1_with_3_mib_block", "block_larger_than_level_1", "stream_signature_in_payload"} <= {c.name for c in cases}
    new, old = _both(units, caps)
    assert not _differences(new, old)
    bad = [(c.name, int(new[0][i]), c.engine) for i, c in enumerate(cases) if new[0][i] != c.engine
           or (c.engine in (OK, WRONG_CRC) and new[3][i] != c.expect) or (c.engine == OK and new[2][i] != c.nbits)]
    assert not bad, bad[:8]
    L = S._lib.lib()
    # a table of 300 entries and the fallback's scratch with 1 MiB to spare (a few dozen slots): most streams take the
    # fallback, the rest run in slices
    small = _run("bzip2_stream", units, caps, max_blocks=300,
                 scratch_bytes=L.swc_bzip2_stream_batch_scratch_bytes(len(units), 1, sum(caps)) + (1 << 20))
    assert not _differences(small, new)


def test_truncations(S, oracle):
    """every byte cut of the small cases, the rest of the stream behind the cut in memory: the old batch's answer, and the
    oracle's status where DESIGN §6 does not let the engine differ"""
    from swcompression_b200.batch import Batch
    trunc = D.truncations()
    buf, offs, lens = H.pack_hostile([t.data for t in trunc], random.Random(91), None, [t.tail for t in trunc])
    caps = np.array([t.spare for t in trunc], dtype=np.uint64)
    res = {}
    for codec in ("bzip2_stream", "bzip2"):
        b = Batch(codec, buf, offs, lens, caps)
        b.run()
        res[codec] = b.results() + (b.outputs(),)
    assert not _differences(res["bzip2_stream"], res["bzip2"])
    st = res["bzip2_stream"][0]
    want = []
    for t in trunc:
        ost = oracle.bzip2_decompress(t.data)[0]
        want.append(UNSUPPORTED if t.oversub else OVERFLOW if ost == UNSUPPORTED else ost)
    assert (st != OK).all() and list(st) == want


@functools.lru_cache(maxsize=None)
def _real_streams():
    """libbzip2 streams of 0, 1 and many blocks at levels 1 and 9: text, random bytes, long runs (blocks larger than a
    slot), and two streams back to back"""
    rng = random.Random(92)
    raws = [b"", b"x", _text(50000, 1), _text(1_500_000, 2), rng.randbytes(700_000), _text(2_300_000, 3),
            b"\0" * 3_000_000, bytes(range(256)) * 20000 + b"\x07" * 2_000_000]
    out = []
    for raw in raws:
        for level in (1, 9):
            out.append((bz2.compress(raw, level), raw))
    out.append((bz2.compress(raws[3], 1) + bz2.compress(raws[2], 9), raws[3]))
    return out


def test_real_streams(S, oracle):
    """the oracle's bytes and consumed bits, the old batch's answer; the concatenation decodes its first stream only"""
    streams = _real_streams()
    units, raws = [s for s, _ in streams], [r for _, r in streams]
    assert max(len(_magics(u)[0]) for u in units) > 20
    new, old = _both(units, [len(r) for r in raws])
    assert not _differences(new, old) and not _oracle_differences(oracle, units, new)
    assert (new[0] == OK).all() and new[3] == raws
    assert new[2][-1] == _magics(bz2.compress(raws[-1], 1))[1] + 80


def test_damage_and_mixed_batch(S, oracle):
    """a flipped block CRC at block k, a flipped combined CRC, a stream cut at a block boundary, a bad header, a stream
    without its end magic, junk bits between two blocks and in front of the end magic: each gives the oracle's status and
    payload, between sound units in one batch"""
    good = [bz2.compress(_text(900_000, 10 + k), 1) for k in range(3)]
    units = []
    for g in good:
        blocks, end = _magics(g)
        units += [g, _flip(g, blocks[3] + 48 + 5), _flip(g, blocks[-1] + 48), _flip(g, end + 48 + 31), g[:blocks[5] // 8],
                  g[:blocks[5] // 8 + 1], b"BZh0" + g[4:], g[:end // 8], _flip(g, blocks[2] + 200),
                  _insert(g, blocks[3], "10110"), _insert(g, end, "01100111")]
    rng = random.Random(93)
    order = list(range(len(units)))
    rng.shuffle(order)
    units = [units[i] for i in order]
    caps = [1_000_000] * len(units)
    new, old = _both(units, caps)
    assert not _differences(new, old) and not _oracle_differences(oracle, units, new)
    assert (new[0] == WRONG_CRC).sum() >= 9 and (new[0] == OK).sum() == 3


def test_overflow_then_rerun(S):
    """capacity one byte short, and half the size: a stream that validated reports its exact size, and the rerun at that
    size succeeds; the old batch's size is a lower bound of it, which stops at the block that crossed the capacity"""
    streams = [s for s in _real_streams() if 0 < len(s[1]) < 3_000_000]
    units, raws = [s for s, _ in streams] * 2, [r for _, r in streams] * 2
    caps = [len(r) - 1 for r in raws[:len(streams)]] + [len(r) // 2 for r in raws[len(streams):]]
    new, old = _both(units, caps)
    assert not _differences(new, old)
    validated = [i for i in range(len(units)) if new[1][i] == len(raws[i])]
    assert len(validated) >= len(units) - 4 and (new[0] == OVERFLOW).all()
    assert sum(old[1][i] < len(raws[i]) for i in validated) >= 4
    redo = _run("bzip2_stream", [units[i] for i in validated], new[1][validated])
    assert (redo[0] == OK).all() and redo[3] == [raws[i] for i in validated]


def test_block_table_too_small(S):
    """a table with room for fewer blocks than the candidates: the units past it take the fallback, with identical results"""
    streams = _real_streams()
    units, caps = [s for s, _ in streams], [len(r) + 5 for _, r in streams]
    full = _run("bzip2_stream", units, caps)
    for mb in (1, 7, 40):
        assert not _differences(_run("bzip2_stream", units, caps, max_blocks=mb), full), mb


def test_one_slot_scratch(S):
    """a scratch with room for one slot decodes one block per slice with identical results (the fourth stream no longer fits
    the fallback behind the first three, so it skips the block stage and the fallback decodes it); a unit whose fallback
    scratch does not fit reports SWC_ERR_UNSUPPORTED and leaves its region untouched, a damaged multi-block stream included"""
    import torch
    from swcompression_b200.batch import Batch
    L = S._lib.lib()
    damaged = bz2.compress(_text(600_000, 24), 1)
    damaged = _flip(damaged, _magics(damaged)[0][3] + 48 + 7)
    units = [bz2.compress(_text(600_000, 20 + k), 1 + 8 * (k % 2)) for k in range(4)] + [b"BZh9\x31\x41", b"notbzip2", damaged]
    caps = [600_000] * 4 + [100, 10_000_000, 3_000_000]
    n, mb = len(units), 40
    one = L.swc_bzip2_stream_batch_scratch_bytes(n, mb, 0) - (mb - 1) * _slot_bytes(L)
    full = _run("bzip2_stream", units, caps, max_blocks=mb)
    assert full[0][6] == WRONG_CRC and (full[0][:4] == OK).all()
    b = Batch.from_units("bzip2_stream", units, np.asarray(caps, dtype=np.uint64), max_blocks=mb, scratch_bytes=one)
    assert b.d_scratch.numel() == one
    b.d_out.fill_(H.SENTINEL)
    b.run()
    st, ln, used = b.results()
    outs = b.outputs()
    assert not _differences((st[:5], ln[:5], used[:5], outs[:5]), tuple(x[:5] for x in full))
    host = b.d_out.cpu().numpy()
    for i in (5, 6):
        assert st[i] == UNSUPPORTED and ln[i] == 0 and used[i] == 0 and full[0][i] != UNSUPPORTED, i
        o = int(b.h_out_off[i])
        assert (host[o:o + caps[i]] == H.SENTINEL).all(), i
    # less than the tables and one slot is refused
    with pytest.raises(RuntimeError):
        Batch.from_units("bzip2_stream", units, np.asarray(caps, dtype=np.uint64), max_blocks=mb, scratch_bytes=one - 256).run()
    torch.cuda.synchronize()


def test_library_count_with_caller_scratch(S, oracle):
    """max_blocks=None with a caller scratch of swc_bzip2_stream_batch_scratch_bytes(n, 0, sum of out_cap): the library counts
    the candidates, keeps the table to what the scratch holds beside every unit's fallback, and every unit gets its exact
    status: a stream of more than 32 blocks alone at a capacity below one slot's fallback, a damaged one, and a mixed batch"""
    raw = _text(4_000_000, 50)
    s40 = bz2.compress(raw, 1)
    blocks = _magics(s40)[0]
    assert len(blocks) > 32
    d40 = _flip(s40, blocks[20] + 48 + 3)
    cases = [([s40], [1 << 20]), ([d40], [len(raw)]), ([s40], [len(raw)]),
             ([s40, d40, bz2.compress(raw[:2_000_000], 9), b"BZh9", s40[:len(s40) // 2]], [len(raw), len(raw), 2_000_000, 100, len(raw)])]
    for k, (units, caps) in enumerate(cases):
        new = _run("bzip2_stream", units, caps, scratch_bytes=1 << 50)      # the Batch caps it at scratch_bytes(n, 0, ...)
        old = _run("bzip2", units, caps)
        assert not _differences(new, old) and not (new[0] == UNSUPPORTED).any(), (k, list(new[0]), list(old[0]))
        if k:                                                                 # every capacity holds the whole output
            assert not _oracle_differences(oracle, units, new), k
    assert list(new[0][:2]) == [OK, WRONG_CRC]
    assert not _differences(_run("bzip2_stream", units, caps), new)           # the library's pool


def _hostile(units, tails, caps_of, rng, codec, max_blocks=0):
    import torch
    from swcompression_b200 import _lib
    out_off, out_cap, total = H.fenced_layout(caps_of, 1 << 17)
    buf, offs, lens = H.pack_hostile(units, rng, None, tails)
    n = len(units)
    d_in, d_off, d_len, d_oo, d_oc = _dev(buf), _dev(offs), _dev(lens), _dev(out_off), _dev(out_cap)
    d_out = torch.full((total,), H.SENTINEL, dtype=torch.uint8, device="cuda")
    d_ln = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_used = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    args = (_p(d_in), _p(d_off), _p(d_len), _p(d_out), _p(d_oo), _p(d_oc), _p(d_ln), _p(d_used), _p(d_st), n)
    if codec == "bzip2":
        assert L.swc_bzip2_decompress_batch(*args, _stream()) == 0
    else:
        assert L.swc_bzip2_stream_decompress_batch(*args, max_blocks, None, 0, _stream()) == 0
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    outs = [bytes(out[int(o):int(o) + int(c)]) for o, c in zip(out_off, out_cap)]
    ln = d_ln.cpu().numpy()
    return (d_st.cpu().numpy(), ln, d_used.cpu().numpy(), [o[:int(l)] for o, l in zip(outs, ln)]), H.fence_violations(out, out_off, out_cap)


def test_hostile_layout(S):
    """the bzip2 layout set of tests/helpers.py plus multi-block streams: units at every start residue and back to back, cut
    streams followed by their rest, capacities exact, short and long between sentinel bytes that must stay intact"""
    units = H.LAYOUT_SETS["bzip2"][1]()
    units += [H.LayoutUnit(bz2.compress(_text(400_000 + 1000 * k, 30 + k), 1), raw=_text(400_000 + 1000 * k, 30 + k)) for k in range(6)]
    data, tails = [u.data for u in units], [u.tail for u in units]
    sizes = [len(u.raw) if u.raw is not None else None for u in units]
    new, fence_new = _hostile(data, tails, sizes, random.Random(94), "bzip2_stream")
    old, fence_old = _hostile(data, tails, sizes, random.Random(94), "bzip2")
    assert fence_new.size == 0 and fence_old.size == 0, fence_new[:8]
    assert not _differences(new, old)
    assert (new[0] == OVERFLOW).sum() > 5 and (new[0] == OK).sum() > 10
    tbl, fence_tbl = _hostile(data, tails, sizes, random.Random(94), "bzip2_stream", max_blocks=25)
    assert fence_tbl.size == 0 and not _differences(tbl, new)


def test_graph_capture(S):
    """with caller scratch and max_blocks > 0 the call reads nothing back and allocates nothing: captured into a CUDA graph,
    the results stay untouched until the replay; replayed on new inputs of the same shape, they equal an eager run's"""
    import torch
    from swcompression_b200.batch import Batch
    ra = [_text(200_000 + 50_000 * (k % 5), 40 + k) for k in range(12)]
    rb = [_text(210_000 + 40_000 * (k % 4), 60 + k) for k in range(12)]
    sa = [bz2.compress(r, 1 + (k % 2) * 8) for k, r in enumerate(ra)]
    sb = [bz2.compress(r, 1 + (k % 3 == 0) * 8) for k, r in enumerate(rb)]
    sb[5] = _flip(sb[5], _magics(sb[5])[0][1] + 48)                 # one damaged unit takes the fallback on the replay
    slot = [(max(len(x), len(y)) + 15) // 16 * 16 for x, y in zip(sa, sb)]
    offs = np.concatenate(([0], np.cumsum(slot)[:-1])).astype(np.uint64)
    pack = lambda ss: np.frombuffer(b"".join(s + b"\0" * (w - len(s)) for s, w in zip(ss, slot)) + b"\0" * 64, dtype=np.uint8).copy()
    caps = np.array([450_000] * 12, dtype=np.uint64)
    mb = sum(len(_magics(s)[0]) for s in sa + sb) + 7
    b = Batch("bzip2_stream", pack(sa), offs, np.array([len(s) for s in sa], dtype=np.uint64), caps, max_blocks=mb)
    b.run()
    st0, _, _ = b.results()
    assert (st0 == OK).all() and b.outputs() == ra
    b.d_status.fill_(-1); b.d_out_len.zero_(); b.d_consumed.zero_(); b.d_out.zero_()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            b.run()
    torch.cuda.synchronize()
    assert (b.d_status.cpu().numpy() == -1).all()
    b.d_in.copy_(torch.from_numpy(pack(sb)))
    b.d_in_len.copy_(torch.from_numpy(np.array([len(x) for x in sb], dtype=np.int64)))
    g.replay()
    st1, ln1, used1 = b.results()
    eager = _run("bzip2_stream", sb, caps)
    assert (st1 == eager[0]).all() and (ln1 == eager[1]).all() and (used1 == eager[2]).all() and b.outputs() == eager[3]
    assert st1[5] == WRONG_CRC and (np.delete(st1, 5) == OK).all()
